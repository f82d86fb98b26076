"""Weight gradient on wgmma (csrc/wgrad_wgmma.cuh: operands gathered K-major, pixel-range split, red.add epilogue) against
an fp64 PyTorch oracle — every ResNet18 site, the VAE / CPC sites (4x4 stride 2, dilated, channel counts that are not
multiples of 32), odd geometries (3x3 latent grid, batch not a multiple of the pixel box) and the in-place
accumulation into a gradient buffer.  Sites: the ResNet18, VAE and CPC convolutions of the original models."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402

DEV = torch.device("cuda", 0)

# B, H, Ci, Co, k, stride, pad, dil
SITES = [
    (128, 32, 4, 64, 3, 1, 1, 1),       # stem (3 channels padded to 4)
    (128, 32, 64, 64, 3, 1, 1, 1),      # layer1
    (128, 32, 64, 128, 3, 2, 1, 1),     # layer2.0.conv1
    (128, 16, 128, 128, 3, 1, 1, 1),    # layer2
    (128, 32, 64, 128, 1, 2, 0, 1),     # layer2.0.shortcut
    (128, 16, 128, 256, 3, 2, 1, 1),    # layer3.0.conv1
    (128, 8, 256, 256, 3, 1, 1, 1),     # layer3
    (128, 16, 128, 256, 1, 2, 0, 1),    # layer3.0.shortcut
    (128, 8, 256, 512, 3, 2, 1, 1),     # layer4.0.conv1
    (128, 4, 512, 512, 3, 1, 1, 1),     # layer4
    (128, 8, 256, 512, 1, 2, 0, 1),     # layer4.0.shortcut
    (128, 32, 4, 12, 4, 2, 1, 1), (128, 16, 12, 24, 4, 2, 1, 1), (128, 8, 24, 48, 4, 2, 1, 1), (128, 4, 48, 96, 4, 2, 1, 1),   # VAE
    (96, 32, 8, 8, 4, 2, 3, 2), (96, 32, 8, 8, 4, 2, 24, 16), (96, 16, 40, 64, 4, 2, 1, 1), (96, 4, 128, 256, 4, 2, 1, 1),     # CPC encoder
    (37, 3, 64, 16, 2, 1, 1, 1), (37, 4, 16, 32, 2, 1, 0, 1), (37, 3, 256, 32, 1, 1, 0, 1),                                     # CPC latent grid
    (5, 6, 20, 12, 3, 1, 1, 1),         # nothing is a power of two
]


def _oracle(x, dy, w_shape, s, p, d):
    x64, dy64 = x.double(), dy.double()
    w = torch.zeros(w_shape, dtype=torch.float64, device=DEV)
    return torch.ops.aten.convolution_backward(dy64, x64, w, None, [s, s], [p, p], [d, d], False, [0, 0], 1, [False, True, False])[1]


@pytest.mark.parametrize("B,H,Ci,Co,k,s,p,d", SITES)
def test_wgrad_matches_fp64_oracle(B, H, Ci, Co, k, s, p, d):
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + H * 10 + Ci + Co + k + d)
    Ho = (H + 2 * p - d * (k - 1) - 1) // s + 1
    xn = torch.randn(B, H, H, Ci, device=DEV, generator=g)
    dyn = torch.randn(B, Ho, Ho, Co, device=DEV, generator=g)
    assert cuda_ops.conv_wgrad_supported(xn, dyn, s)
    dw = cuda_ops.conv_wgrad(xn, dyn, k, k, Ci, s, p, d)                      # logical [Co, Ci, k, k]
    ref = _oracle(xn.permute(0, 3, 1, 2), dyn.permute(0, 3, 1, 2), (Co, Ci, k, k), s, p, d)
    assert dw.shape == ref.shape
    err = float((dw.double() - ref).abs().max() / ref.abs().max())
    assert err < 3e-3, err                                                     # tf32 products, fp32 accumulation


def test_wgrad_channel_padded_input_and_inplace_accumulation():
    """Stem: x carries 4 channels (3 + TMA padding), dW has 3; with ``accumulate_into_grad`` the kernel adds to the
    parameter's gradient buffer (KRSC memory, like the channels-last arena) and returns None."""
    g = torch.Generator(device=DEV).manual_seed(5)
    B, H, Co = 64, 32, 64
    x3 = torch.randn(B, H, H, 3, device=DEV, generator=g)
    xn = torch.nn.functional.pad(x3, (0, 1))
    dyn = torch.randn(B, H, H, Co, device=DEV, generator=g)
    ref = _oracle(x3.permute(0, 3, 1, 2), dyn.permute(0, 3, 1, 2), (Co, 3, 3, 3), 1, 1, 1)
    dw = cuda_ops.conv_wgrad(xn, dyn, 3, 3, 3, 1, 1, 1)
    assert float((dw.double() - ref).abs().max() / ref.abs().max()) < 3e-3
    w = torch.nn.Parameter(torch.zeros(Co, 3, 3, 3, device=DEV).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2))
    w.grad = torch.ones(Co, 3, 3, 3, device=DEV).contiguous().permute(0, 3, 1, 2)       # KRSC memory, pre-filled with ones
    with cuda_ops.accumulate_into_grad():
        out = cuda_ops.conv_wgrad(xn, dyn, 3, 3, 3, 1, 1, 1, w)
    assert out is None
    assert float((w.grad.double() - 1.0 - ref).abs().max() / ref.abs().max()) < 3e-3
    assert cuda_ops.conv_wgrad(xn, dyn, 3, 3, 3, 1, 1, 1, w) is not None          # outside the context: returned, .grad untouched
