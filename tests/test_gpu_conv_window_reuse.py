"""The window-reuse main loop of the pixel-major wgmma convolution (csrc/igemm_wgmma.cuh: igemm_wgmma_pix_kernel with WIN_KH = 3)
against a float64 oracle: forward with BatchNorm statistics, plain store and the stride-1 data gradient, at batches
1, 5 and 128, on the ResNet18 layer-1 shape (64 channels, 32 x 32), 16 x 16 maps (one tile per image) and a 24 x 32 map whose
middle tile takes its halo rows from the tiles above and below; and its agreement with the per-tap loop.  Run on an H100:
``python -m pytest tests -m gpu``."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402

DEV = torch.device("cuda", 0)
PIXEL, PIXEL_PERTAP = 1, 2


@pytest.fixture(autouse=True)
def _exact_reference_math():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def oracle(x, w, p):
    return F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, 1, p).permute(0, 2, 3, 1)


def _marked(t):
    """Large offsets on the first / last row and column of every image, distinct per edge and per image: a halo row read from
    the wrong place, from a neighbouring image, or a missing zero fill changes the result well above the tolerance.  Images
    2i and 2i + 1 carry opposite offsets, so over a batch they cancel and the channel sums keep the zero mean the statistics
    tolerance assumes (a same-sign offset on every image turns the tf32 rounding of the weights into a bias of the sums)."""
    B = t.shape[0]
    n = torch.arange(B, device=t.device, dtype=t.dtype)
    scale = ((1.0 - 2.0 * (n % 2)) * (1.0 + 0.01 * torch.div(n, 2, rounding_mode="floor"))).view(B, 1, 1)
    t[:, 0] += 3.0 * scale
    t[:, -1] -= 5.0 * scale
    t[:, :, 0] += 7.0 * scale
    t[:, :, -1] -= 2.0 * scale
    return t


# (H, W, C): layer 1 (64 channels, 32 x 32: four 8-row tiles per image), 16 x 16 (one 16-row tile per image, 2 KB image rows),
# and 24 x 32 (three 8-row tiles per image)
SHAPES = [(32, 32, 64), (16, 16, 64), (24, 32, 64)]
BATCHES = [1, 5, 128]


def _inputs(B, H, W, C):
    g = torch.Generator(device=DEV).manual_seed(B * H + W + C)
    x = _marked(torch.randn(B, H, W, C, device=DEV, generator=g))
    w = torch.randn(C, 3, 3, C, device=DEV, generator=g) / math.sqrt(9 * C)
    return x, w


def test_window_reuse_selection():
    q = cuda_ops.ext().conv_window_reuse
    for H, W, C in SHAPES:
        assert q(H, W, C, C, 3, 1, 1)
    assert not q(16, 16, 128, 128, 3, 1, 1)      # layer 2 (128 channels): the per-tap loop
    assert not q(16, 16, 64, 128, 3, 2, 1)       # stride 2
    assert not q(16, 16, 64, 128, 1, 2, 1)       # 1 x 1 shortcut
    assert not q(32, 32, 4, 64, 3, 1, 1)         # the tap-packed stem (C_in 4)
    assert not q(8, 8, 64, 64, 3, 1, 1)          # a 256-pixel tile spans four images
    assert not q(32, 32, 64, 64, 3, 1, 2)        # dilation
    assert not q(8, 8, 256, 256, 3, 1, 1)        # C_out 256: row-major tiles


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,W,C", SHAPES)
def test_forward_with_batchnorm_statistics(B, H, W, C):
    x, w = _inputs(B, H, W, C)
    stats = torch.zeros(2 * C, device=DEV)
    y = cuda_ops.ext().conv2d_nhwc(x, w, stats, 1, 1, 1, PIXEL)
    ref = oracle(x, w, 1).float()
    assert y.shape == ref.shape
    assert rel_err(y, ref) < 3e-3
    flat = ref.reshape(-1, C)
    torch.testing.assert_close(stats[:C], flat.sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(flat.shape[0]))
    torch.testing.assert_close(stats[C:], (flat * flat).sum(0), rtol=5e-3, atol=1e-2)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,W,C", SHAPES)
def test_plain_store(B, H, W, C):
    x, w = _inputs(B, H, W, C)
    y = cuda_ops.ext().conv2d_nhwc(x, w, None, 1, 1, 1, PIXEL)
    assert rel_err(y, oracle(x, w, 1).float()) < 3e-3


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,W,C", SHAPES)
def test_stride1_data_gradient(B, H, W, C):
    """dx of a 3 x 3 stride-1 convolution = conv(dy, rotated and transposed filter), as the training backward runs it."""
    e = cuda_ops.ext()
    x, w = _inputs(B, H, W, C)
    dy = _marked(torch.randn(B, H, W, C, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B + H + W)))
    dx = e.conv2d_nhwc(dy, e.weight_flip(w), None, 1, 1, 1, PIXEL)
    ref = torch.ops.aten.convolution_backward(
        dy.permute(0, 3, 1, 2).double(), x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None,
        [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])[0].permute(0, 2, 3, 1)
    assert rel_err(dx, ref.float()) < 3e-3


@pytest.mark.parametrize("H,W,C", SHAPES)
def test_window_reuse_agrees_with_per_tap_loop_at_batch_128(H, W, C):
    e = cuda_ops.ext()
    x, w = _inputs(128, H, W, C)
    st_tap, st_win = torch.zeros(2 * C, device=DEV), torch.zeros(2 * C, device=DEV)
    y_tap = e.conv2d_nhwc(x, w, st_tap, 1, 1, 1, PIXEL_PERTAP)
    y_win = e.conv2d_nhwc(x, w, st_win, 1, 1, 1, PIXEL)
    assert rel_err(y_win, y_tap) < 1e-4        # same tf32 products, fp32 sums in another order
    torch.testing.assert_close(st_win, st_tap, rtol=1e-4, atol=1e-2)
