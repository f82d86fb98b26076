"""The window-reuse decomposition of the pixel-major convolution kernel (ops/conv_math.py: window_reuse_conv_oracle) against
F.conv2d, on CPU: one box of tile rows + kh - 1 input rows per filter column serves all kh filter rows."""
import pytest
import torch
import torch.nn.functional as F

from federated_pytorch_test_b200.ops import conv_math


def _inputs(N, H, W, Ci, Co, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, Ci, generator=g, dtype=torch.float64)
    # large, distinct first / last rows and columns: a halo row taken from the wrong place or a missing zero fill shows
    x[:, 0] += 100.0
    x[:, -1] -= 300.0
    x[:, :, 0] += 1000.0
    x[:, :, -1] -= 3000.0
    w = torch.randn(Co, k, k, Ci, generator=g, dtype=torch.float64)
    return x, w


# (H, W, tile rows): 24 x 16 with 8-row tiles has a top, a middle and a bottom tile; 32 x 32 with 8-row tiles is layer 1 of
# ResNet18 (256-pixel tiles); 16 x 16 with 16-row tiles is layer 2 (one tile = the whole image, both edges at once)
@pytest.mark.parametrize("H,W,rows", [(24, 16, 8), (32, 32, 8), (16, 16, 16)])
@pytest.mark.parametrize("pad", [1, 0])
def test_window_reuse_equals_conv2d(H, W, rows, pad):
    N, Ci, Co, k = 2, 64, 8, 3
    if (H + 2 * pad - k + 1) % rows:
        rows = H + 2 * pad - k + 1          # pad 0 shrinks the map: one tile of all its rows
    x, w = _inputs(N, H, W, Ci, Co, k, seed=H * W + rows + pad)
    y = conv_math.window_reuse_conv_oracle(x, w, pad, rows)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), None, 1, pad).permute(0, 2, 3, 1)
    assert y.shape == ref.shape
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-9)


def test_window_reuse_middle_tile_reads_neighbouring_rows():
    """The middle tile's halo rows are the last row of the tile above and the first row of the tile below."""
    x, w = _inputs(1, 24, 16, 32, 4, 3, seed=7)
    y = conv_math.window_reuse_conv_oracle(x, w, 1, 8)
    x2 = x.clone()
    x2[:, 7] = 0.0                           # the row above the middle tile (rows 8 .. 15)
    y2 = conv_math.window_reuse_conv_oracle(x2, w, 1, 8)
    changed = (y - y2).abs().amax(dim=(0, 2, 3)) > 0
    assert changed.nonzero().flatten().tolist() == [6, 7, 8]
