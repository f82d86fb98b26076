"""Hand-written fp32 kernels of csrc/aux_kernels.cu against plain PyTorch (fp32 / fp64) oracles: dense layers forward +
both gradients, activation-backward + bias sums, 2x2 max-pool (NCHW and NHWC), evaluation argmax/count, fused InfoNCE
(vs the reference's P^2 loop at small P), Gaussian-NLL rows of the VAE-CL cost, direct small convolutions (Net), and
the model-level consequences: Net / Net2 / VAE / VAE-CL / CPC forward+backward on the fast path vs the ATen path, and
"no library GEMM / convolution kernel in a training step" for ResNet18, the VAE and Net."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200 import models  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops, losses  # noqa: E402
from federated_pytorch_test_b200.ops import functional as FX  # noqa: E402

DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _exact_reference_math():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    FX.set_fast_path(True)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_err(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-20))


@pytest.mark.parametrize("M,N,K", [(128, 10, 512), (128, 120, 400), (128, 84, 120), (1280, 128, 394), (37, 3, 5), (256, 384, 10)])
@pytest.mark.parametrize("act", [False, True])
def test_linear_f32_forward_and_gradients(M, N, K, act):
    torch.manual_seed(M + N + K)
    lin = nn.Linear(K, N).to(DEV)
    x = torch.randn(M, K, device=DEV, requires_grad=True)
    assert cuda_ops.linear_act_supported(x, lin)
    y = cuda_ops.linear_act(x, lin, act)
    ref = F.linear(x, lin.weight, lin.bias)
    ref = F.elu(ref) if act else ref
    torch.testing.assert_close(y, ref, rtol=2e-5, atol=2e-5)
    g = torch.randn_like(ref)
    gx, gw, gb = torch.autograd.grad(y, (x, lin.weight, lin.bias), g)
    rx, rw, rb = torch.autograd.grad(ref, (x, lin.weight, lin.bias), g)
    assert rel_err(gx, rx) < 1e-4 and rel_err(gw, rw) < 1e-4 and rel_err(gb, rb) < 1e-4
    # in-place accumulation into gradient buffers (what the engine's backward uses)
    lin.weight.grad, lin.bias.grad = torch.ones_like(lin.weight), torch.ones_like(lin.bias)
    with cuda_ops.accumulate_into_grad():
        cuda_ops.linear_act(x, lin, act).backward(g)
    assert rel_err(lin.weight.grad - 1, rw) < 1e-4 and rel_err(lin.bias.grad - 1, rb) < 1e-4


@pytest.mark.parametrize("M,C", [(4096, 3), (1000, 12), (777, 96), (64, 1024), (131072, 8)])
def test_act_bwd_bias(M, C):
    g = torch.Generator(device=DEV).manual_seed(M + C)
    z = torch.randn(M, C, device=DEV, generator=g)
    out = F.elu(z)
    dout = torch.randn(M, C, device=DEV, generator=g)
    dz, db = cuda_ops._act_bwd_bias(dout, out, True, True)
    ref = dout * torch.where(z > 0, torch.ones_like(z), torch.exp(z))
    torch.testing.assert_close(dz, ref, rtol=1e-4, atol=1e-5)
    assert rel_err(db, ref.double().sum(0)) < 1e-4
    dz2, db2 = cuda_ops._act_bwd_bias(dout, None, False, True)
    assert dz2.data_ptr() == dout.data_ptr() and rel_err(db2, dout.double().sum(0)) < 1e-4


@pytest.mark.parametrize("shape", [(8, 6, 28, 28), (5, 16, 10, 10), (3, 7, 9, 11)])
@pytest.mark.parametrize("nhwc", [False, True])
def test_maxpool2x2(shape, nhwc):
    torch.manual_seed(sum(shape))
    x = torch.randn(*shape, device=DEV)
    if nhwc:
        x = x.contiguous(memory_format=torch.channels_last)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    ya = cuda_ops.max_pool2x2(xa)
    yb = F.max_pool2d(xb, 2, 2)
    torch.testing.assert_close(ya, yb, rtol=0, atol=0)
    g = torch.randn_like(yb)
    ya.backward(g)
    yb.backward(g)
    torch.testing.assert_close(xa.grad, xb.grad, rtol=0, atol=0)


def test_argmax_count():
    g = torch.Generator(device=DEV).manual_seed(1)
    counter = torch.zeros(2, dtype=torch.int64, device=DEV)
    want = 0
    for B in (128, 16, 1000):
        logits = torch.randn(B, 10, device=DEV, generator=g)
        labels = torch.randint(0, 10, (B,), device=DEV, generator=g)
        cuda_ops.argmax_count(logits, labels, counter)
        want += int((logits.argmax(1) == labels).sum())
    assert counter.tolist() == [want, 128 + 16 + 1000]


@pytest.mark.parametrize("B,C,px,py", [(16, 8, 3, 3), (128, 32, 3, 3), (8, 16, 4, 5), (4, 4, 1, 2)])
def test_info_nce_fused_vs_reference_loop(B, C, px, py):
    torch.manual_seed(B + C + px)
    z = torch.randn(B, C, px, py, device=DEV, requires_grad=True)
    zh = (0.5 * z.detach() + torch.randn(B, C, px, py, device=DEV)).requires_grad_()
    assert cuda_ops.info_nce_supported(z)
    la = losses.info_nce(z, zh)
    lb = losses.info_nce_reference(z.double(), zh.double())           # the reference's P^2 dot-product loop
    assert float(la) == pytest.approx(float(lb), rel=2e-4)
    ga = torch.autograd.grad(la, (z, zh))
    zd, zhd = z.detach().double().requires_grad_(), zh.detach().double().requires_grad_()
    FX.set_fast_path(False)
    gb = torch.autograd.grad(losses.info_nce(zd, zhd), (zd, zhd))
    FX.set_fast_path(True)
    for u, v in zip(ga, gb):
        assert rel_err(u, v) < 2e-3
    la2 = losses.info_nce(z, zh)                                       # the scratch cleaned itself
    assert float(la2) == pytest.approx(float(la), rel=1e-6)


def test_gauss_nll_rows_and_vae_cl_loss():
    torch.manual_seed(3)
    Kc, B, L = 4, 16, 8
    x = torch.rand(B, 3, 32, 32, device=DEV)
    mu = torch.randn(Kc, B, 3, 32, 32, device=DEV, requires_grad=True)
    s2 = (torch.rand(Kc, B, 3, 32, 32, device=DEV) + 0.3).requires_grad_()
    rows = cuda_ops.gauss_nll_rows(x, mu, s2)
    ref = ((x.unsqueeze(0) - mu).pow(2) / (2 * s2) + 0.5 * torch.log(s2 * 2 * math.pi)).flatten(2).sum(-1)
    torch.testing.assert_close(rows, ref, rtol=2e-4, atol=1e-2)
    w = torch.randn_like(ref)
    ga = torch.autograd.grad(rows, (mu, s2), w)
    gb = torch.autograd.grad(ref, (mu, s2), w)
    for u, v in zip(ga, gb):
        assert rel_err(u, v) < 1e-3
    # whole VAE-CL loss: fast path vs ATen expression vs the loop oracle
    ek = torch.softmax(torch.randn(B, Kc, device=DEV), 1)
    args = (ek, torch.randn(Kc, B, L, device=DEV), torch.rand(Kc, B, L, device=DEV) + 0.2, torch.randn(Kc, B, L, device=DEV),
            torch.rand(Kc, B, L, device=DEV) + 0.2, mu.detach(), s2.detach(), x)
    fast = losses.vae_cl_loss(*args)
    FX.set_fast_path(False)
    slow = losses.vae_cl_loss(*args)
    FX.set_fast_path(True)
    assert float(fast) == pytest.approx(float(slow), rel=1e-4)
    assert float(fast) == pytest.approx(float(losses.vae_cl_loss_reference(*args)), rel=1e-3)


@pytest.mark.parametrize("B,Ci,H,Co,k,pad,act,pool", [(16, 3, 32, 6, 5, 0, True, True), (16, 6, 14, 16, 5, 0, True, True),
                                                    (8, 3, 32, 32, 3, 0, True, False), (8, 32, 30, 32, 3, 0, True, True),
                                                    (4, 64, 3, 64, 2, 1, True, False), (4, 64, 4, 128, 2, 0, True, False),
                                                    (5, 7, 9, 5, 3, 1, False, False)])
def test_small_direct_conv_forward_backward(B, Ci, H, Co, k, pad, act, pool):
    torch.manual_seed(B + Ci + H + Co)
    conv = nn.Conv2d(Ci, Co, k, padding=pad).to(DEV)
    x = torch.randn(B, Ci, H, H, device=DEV, requires_grad=True)
    assert cuda_ops.smallconv_supported(x, conv)
    y = cuda_ops.small_conv(x, conv, act, pool)
    ref = conv(x)
    ref = F.elu(ref) if act else ref
    ref = F.max_pool2d(ref, 2, 2) if pool else ref
    torch.testing.assert_close(y, ref, rtol=1e-4, atol=1e-5)
    g = torch.randn_like(ref)
    gx, gw, gb = torch.autograd.grad(y, (x, conv.weight, conv.bias), g)
    rx, rw, rb = torch.autograd.grad(ref, (x, conv.weight, conv.bias), g)
    assert rel_err(gx, rx) < 1e-4 and rel_err(gw, rw) < 1e-4 and rel_err(gb, rb) < 1e-4


@pytest.mark.parametrize("B,Ci,H,Co,k,pad,act", [(128, 64, 3, 64, 2, 1, True), (128, 64, 4, 128, 2, 0, True), (16, 256, 3, 64, 2, 1, False),
                                                 (9, 32, 5, 24, 3, 1, True)])
def test_unfold_gemm_conv_forward_backward(B, Ci, H, Co, k, pad, act):
    """2x2 / 3x3 convolutions on the CPC latent grid: im2col rows x fp32 GEMM kernel (true fp32 -> tight tolerance)."""
    torch.manual_seed(B + Ci + H + Co)
    conv = nn.Conv2d(Ci, Co, k, padding=pad, bias=(B != 16)).to(DEV)
    x = torch.randn(B, Ci, H, H, device=DEV, requires_grad=True)
    assert cuda_ops.unfold_conv_supported(x, conv)
    n0 = cuda_ops.launch_count()
    y = cuda_ops.unfold_conv(x, conv, act)
    assert cuda_ops.launch_count() - n0 == 1           # the GEMM kernel (bias + ELU in its epilogue)
    ref = F.conv2d(x.double(), conv.weight.double(), conv.bias.double() if conv.bias is not None else None, 1, pad)
    ref = F.elu(ref) if act else ref
    assert y.shape == ref.shape and rel_err(y.double(), ref) < 1e-5
    g = torch.randn_like(y)
    params = [x, conv.weight] + ([conv.bias] if conv.bias is not None else [])
    for u, v in zip(torch.autograd.grad(y, params, g), torch.autograd.grad(ref, params, g.double())):
        assert rel_err(u.double(), v) < 1e-4


def _twin_grads(factory, inputs, loss_fn, tol, ref_double=False):
    """Same module twice; one stepped on the fast path, one on the ATen path (optionally in fp64: cuDNN's fp32 convolutions
    may still multiply in TF32); compares loss and every parameter gradient."""
    torch.manual_seed(0)
    a = factory().to(DEV)
    b = factory().to(DEV)
    b.load_state_dict(a.state_dict())
    ref_inputs = inputs
    if ref_double:
        b = b.double()
        ref_inputs = tuple(t.double() if t.is_floating_point() else t for t in inputs)
    torch.manual_seed(1)
    FX.set_fast_path(True)
    la = loss_fn(a, *inputs)
    la.backward()
    torch.manual_seed(1)
    FX.set_fast_path(False)
    lb = loss_fn(b, *ref_inputs)
    lb.backward()
    FX.set_fast_path(True)
    assert float(la) == pytest.approx(float(lb), rel=tol)
    errs = {n: rel_err(pa.grad, pb.grad) for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters())}
    bad = {n: e for n, e in errs.items() if not e < 10 * tol}
    assert not bad, "per-parameter gradient errors: %s" % errs


@pytest.mark.parametrize("name", ["Net", "Net1"])
def test_net_fast_path_matches_fp64_oracle(name):
    """Net / Net1 run entirely in true fp32 on the fast path (direct convolutions with ELU + max-pool fused, fp32 dense kernels).
    The input seed is fixed: a max-pool winner that is a near-tie at fp32 resolution may be resolved differently by an fp64
    oracle, which moves one term of a conv weight gradient (~1 % of an entry) — a property of the comparison, not of the kernels
    (the layer-level tests above pin the kernels at 1e-4)."""
    torch.manual_seed(1000)
    x = torch.randn(32, 3, 32, 32, device=DEV)
    y = torch.randint(0, 10, (32,), device=DEV)
    _twin_grads(getattr(models, name), (x, y), lambda m, xx, yy: losses.cross_entropy(m(xx), yy), 1e-4, ref_double=True)


def _l2_err(u, v):
    return float((u.double() - v.double()).norm() / v.double().norm().clamp_min(1e-30))


def test_net2_fast_path_vs_fp64_oracles():
    """Net2's convolutions run on the TF32 tensor cores.  A plain fp64 oracle disagrees with that by MORE than TF32's 2^-11:
    the operand rounding flips a small fraction of the 2x2 max-pool winners and every flip moves one term of the upstream
    gradients, which shows up
    as 2-6 % relative L2 error in the conv weight gradients while everything downstream of the last pool (conv4.bias, fc*) agrees
    to 5e-4.  An oracle that rounds the conv operands to TF32 (round-to-nearest) removes 2/3 of that.  (ATen / cuDNN on this
    image does not take a plain-TF32 path for these shapes — its error against fp64 is 1e-4 — so it is no yardstick either.)
    Bounds here: a wrong tap / layout / missing term would be an O(1) error; the kernels themselves are pinned at 3e-3 by the
    layer-level tests (conv + bias + ELU forward / dgrad / wgrad, NHWC max-pool, dense layers)."""
    from federated_pytorch_test_b200.utils.tf32_oracle import tf32_conv_oracle
    torch.manual_seed(1000)
    x = torch.randn(32, 3, 32, 32, device=DEV)
    y = torch.randint(0, 10, (32,), device=DEV)
    torch.manual_seed(0)
    a = models.Net2().to(DEV)
    FX.set_fast_path(True)
    la = losses.cross_entropy(a(x), y)
    la.backward()
    errs = {}
    for mode in ("fp64", "rna"):
        o = models.Net2().to(DEV)
        o.load_state_dict(a.state_dict())
        o = o.double()
        if mode == "rna":
            tf32_conv_oracle(o, "rna")
        FX.set_fast_path(False)
        lo = losses.cross_entropy(o(x.double()), y)
        lo.backward()
        FX.set_fast_path(True)
        assert float(la) == pytest.approx(float(lo), rel=1e-5)
        errs[mode] = {n: _l2_err(pa.grad, po.grad) for (n, pa), (_, po) in zip(a.named_parameters(), o.named_parameters())}
    print("Net2 gradient L2 errors:", {n: "%.1e (fp64) %.1e (tf32-rna)" % (errs["fp64"][n], errs["rna"][n]) for n in errs["fp64"]})
    for n in errs["fp64"]:
        after_last_pool = n.startswith("fc") or n == "conv4.bias"
        assert errs["fp64"][n] < (2e-3 if after_last_pool else 0.12), (n, errs["fp64"][n])
        assert errs["rna"][n] < (1e-3 if after_last_pool else 0.05), (n, errs["rna"][n])


def test_vae_and_cpc_fast_path_match_aten():
    x = torch.rand(32, 3, 32, 32, device=DEV)

    def vae_loss(m, xx):
        recon, mu, logvar = m(xx)
        return losses.vae_loss(recon, xx, mu, logvar)

    _twin_grads(models.AutoEncoderCNN, (x,), vae_loss, 5e-3)

    def cl_loss(m, xx):
        return losses.vae_cl_loss(*m(xx), xx)

    _twin_grads(lambda: models.AutoEncoderCNNCL(K=4, L=8), (x,), cl_loss, 5e-3)

    patches = torch.randn(8 * 9, 8, 32, 32, device=DEV)

    class CPC(nn.Module):
        def __init__(self):
            super().__init__()
            self.enc, self.ctx, self.pred = models.EncoderCNN(64), models.ContextgenCNN(64), models.PredictorCNN(64, 16)

        def forward(self, p):
            lat = self.enc(p).reshape(8, 3, 3, -1).permute(0, 3, 1, 2).contiguous()
            return self.pred(lat, self.ctx(lat))

    _twin_grads(CPC, (patches,), lambda m, p: losses.info_nce(*m(p)), 1e-2)


def _kernel_names(step):
    step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


_LIB = ("cudnn", "cutlass", "cublas", "sgemm", "xmma", "implicit_gemm", "gemv", "gemmk1")


@pytest.mark.parametrize("name", ["ResNet18", "Net", "AutoEncoderCNN"])
def test_training_step_launches_no_library_gemm_or_convolution(name):
    """The profiler's kernel list of one forward + backward with every parameter trainable (VERDICT r1 next-steps 2, 3)."""
    from federated_pytorch_test_b200.utils.flat import FlatArena

    torch.manual_seed(0)
    net = getattr(models, name)().to(DEV)
    cl = name.startswith("ResNet")
    arena = FlatArena(net, device=DEV, channels_last_weights=cl)
    arena.attach_grads()
    x = torch.rand(64, 3, 32, 32, device=DEV)
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (64,), device=DEV)

    def step():
        arena.zero_grads()
        with cuda_ops.accumulate_into_grad():
            if name == "AutoEncoderCNN":
                recon, mu, logvar = net(x)
                losses.vae_loss(recon, x, mu, logvar).backward()
            else:
                losses.cross_entropy(net(x), y).backward()

    names = _kernel_names(step)
    lib = [n for n in names if any(t in n.lower() for t in _LIB)]
    assert not lib, lib
    assert any("fedb200" in n for n in names)
