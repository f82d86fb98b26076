"""The pixel-major wgmma convolution (csrc/igemm_wgmma.cuh: igemm_wgmma_pix_kernel, C_out 64 / 128 x 256-pixel tiles) against
a float64 oracle on every shape it serves in ResNet18, at batch 128 and at small batches whose last pixel tile is partial,
and the orientation conv2d_nhwc picks by itself.  Run on an H100: ``python -m pytest tests -m gpu``."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402

DEV = torch.device("cuda", 0)
ROW, PIXEL = 0, 1


@pytest.fixture(autouse=True)
def _exact_reference_math():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def oracle(x, w, s, p):
    return F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, s, p).permute(0, 2, 3, 1)


# (H_in, C_in, C_out, k, stride, pad): the stem (4 -> 64, tap packing), layer 1 and 2 convolutions, the layer-2 stride-2
# convolution and 1 x 1 shortcut, and 8 x 8 outputs (four images per 256-pixel tile) for partial last tiles
FWD = [(32, 4, 64, 3, 1, 1), (32, 64, 64, 3, 1, 1), (16, 128, 128, 3, 1, 1), (32, 64, 128, 3, 2, 1), (32, 64, 128, 1, 2, 0),
       (8, 64, 64, 3, 1, 1), (16, 64, 128, 3, 2, 1), (8, 128, 128, 3, 1, 1)]
BATCHES = [128, 5, 13]


def _inputs(B, H, Ci, Co, k):
    g = torch.Generator(device=DEV).manual_seed(B * H + Ci + Co + k)
    x = torch.randn(B, H, H, Ci, device=DEV, generator=g)
    w = torch.randn(Co, k, k, Ci, device=DEV, generator=g) / math.sqrt(k * k * Ci)
    return x, w


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,Ci,Co,k,s,p", FWD)
def test_forward_with_batchnorm_statistics(B, H, Ci, Co, k, s, p):
    x, w = _inputs(B, H, Ci, Co, k)
    stats = torch.zeros(2 * Co, device=DEV)
    y = cuda_ops.ext().conv2d_nhwc(x, w, stats, s, p, 1, PIXEL)
    ref = oracle(x, w, s, p).float()
    assert y.shape == ref.shape
    assert rel_err(y, ref) < 3e-3
    flat = ref.reshape(-1, Co)
    torch.testing.assert_close(stats[:Co], flat.sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(flat.shape[0]))
    torch.testing.assert_close(stats[Co:], (flat * flat).sum(0), rtol=5e-3, atol=1e-2)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,Ci,Co,k,s,p", FWD)
def test_plain_store(B, H, Ci, Co, k, s, p):
    x, w = _inputs(B, H, Ci, Co, k)
    y = cuda_ops.ext().conv2d_nhwc(x, w, None, s, p, 1, PIXEL)
    assert rel_err(y, oracle(x, w, s, p).float()) < 3e-3


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,C", [(32, 64), (16, 128), (8, 64), (8, 128)])
def test_stride1_data_gradient(B, H, C):
    """dx of a 3 x 3 stride-1 convolution = conv(dy, rotated and transposed filter), as the training backward runs it."""
    e = cuda_ops.ext()
    g = torch.Generator(device=DEV).manual_seed(B + H + C)
    x = torch.randn(B, H, H, C, device=DEV, generator=g)
    w = torch.randn(C, 3, 3, C, device=DEV, generator=g) / math.sqrt(9 * C)
    dy = torch.randn(B, H, H, C, device=DEV, generator=g)
    dx = e.conv2d_nhwc(dy, e.weight_flip(w), None, 1, 1, 1, PIXEL)
    ref = torch.ops.aten.convolution_backward(
        dy.permute(0, 3, 1, 2).double(), x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None,
        [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])[0].permute(0, 2, 3, 1)
    assert rel_err(dx, ref.float()) < 3e-3


def test_both_orientations_agree_at_batch_128():
    e = cuda_ops.ext()
    x, w = _inputs(128, 32, 64, 64, 3)
    st_row, st_pix = torch.zeros(128, device=DEV), torch.zeros(128, device=DEV)
    y_row = e.conv2d_nhwc(x, w, st_row, 1, 1, 1, ROW)
    y_pix = e.conv2d_nhwc(x, w, st_pix, 1, 1, 1, PIXEL)
    assert rel_err(y_pix, y_row) < 1e-4        # same tf32 products, fp32 sums in another order
    torch.testing.assert_close(st_pix, st_row, rtol=1e-4, atol=1e-2)


def test_orientation_selection(monkeypatch):
    monkeypatch.delenv("FEDB200_BLOCK_N", raising=False)
    pick = cuda_ops.ext().conv_orientation
    # ResNet18 at batch 128: stem, layer 1 forward / data gradient, layer 2 forward (stride 1 and 2, shortcut) / data gradient
    assert pick(128, 32, 32, 64, 1) == PIXEL
    assert pick(128, 16, 16, 128, 1) == PIXEL
    assert pick(128, 16, 16, 128, 2) == PIXEL
    # layers 3 and 4 (C_out 256 / 512), and grids of 256-pixel tiles too short to fill the GPU
    assert pick(128, 8, 8, 256, 1) == ROW
    assert pick(128, 4, 4, 512, 1) == ROW
    assert pick(5, 32, 32, 64, 1) == ROW
    assert pick(20, 16, 16, 128, 1) == ROW
    monkeypatch.setenv("FEDB200_BLOCK_N", "64")       # a forced row-major tile width keeps the row-major kernel
    assert pick(128, 32, 32, 64, 1) == ROW


def test_pixel_major_rejects_unserved_shapes():
    e = cuda_ops.ext()
    x, w = _inputs(4, 8, 256, 256, 3)
    with pytest.raises(RuntimeError, match="pixel-major"):
        e.conv2d_nhwc(x, w, None, 1, 1, 1, PIXEL)
