"""Stride-2 convolution data gradient as ONE stride-1 convolution + a pixel shuffle (SURVEY G1, dgrad).

For ``y = conv(x, W)`` with stride 2 (3x3 / pad 1 or 1x1 / pad 0, reference sites ``src/simple_models.py:137-147``)

    dx[n, 2i+ph, 2j+pw, ci] = sum_{dr,ds in {0,1}} sum_co dy[n, i+dr, j+ds, co] * Wp[(ph,pw,ci), dr, ds, co]

i.e. every output *phase* (ph, pw) is a small stride-1 convolution of ``dy`` anchored at the top-left pixel, and all
four phases together are one 2x2 convolution with ``4*Ci`` output channels whose filter ``Wp`` holds the original taps
(zeros where a phase has no tap):   row phase 0 <- filter row 1 at dr=0;  row phase 1 <- filter row 2 at dr=0 and
filter row 0 at dr=1 (same for columns).  The result ``[N, Ho, Wo, 2, 2, Ci]`` is interleaved into ``[N, 2Ho, 2Wo, Ci]``.

Why: a strided data gradient as a library call (cuDNN ``strided_dgrad``) is a slow kernel, while one stride-1 implicit
GEMM over the phase-packed filter keeps the tensor cores busy; 7/16 of the packed filter is zero padding, which is cheaper
than four launches.

Everything here is plain PyTorch (runs on CPU for the tests); the convolution itself is injected.
"""
from __future__ import annotations

from typing import Callable

import torch
import torch.nn.functional as F

# (phase, d) -> original filter index along that axis for k=3, pad=1, stride=2; (0, 1) has no tap
_TAP3 = {(0, 0): 1, (1, 0): 2, (1, 1): 0}


def _tap_index_table(k: int) -> torch.Tensor:
    """[2,2,2,2] (ph, pw, dr, ds) -> flat tap index r*k+s into the KRSC filter, k*k = "zero tap"."""
    zero = k * k
    idx = torch.full((2, 2, 2, 2), zero, dtype=torch.long)
    for ph in (0, 1):
        for pw in (0, 1):
            for dr in (0, 1):
                for ds in (0, 1):
                    if k == 3:
                        r, s = _TAP3.get((ph, dr)), _TAP3.get((pw, ds))
                    else:  # k == 1, pad 0: only phase (0,0) at (dr,ds) = (0,0)
                        r = 0 if (ph == 0 and dr == 0) else None
                        s = 0 if (pw == 0 and ds == 0) else None
                    if r is not None and s is not None:
                        idx[ph, pw, dr, ds] = r * k + s
    return idx


def pack_dgrad_s2_weight(w_krsc: torch.Tensor) -> torch.Tensor:
    """``[Co, k, k, Ci]`` (k in {1, 3}) -> ``[4*Ci, 2, 2, Co]`` filter of the equivalent stride-1 convolution over dy."""
    Co, kh, kw, Ci = w_krsc.shape
    assert kh == kw and kh in (1, 3), "stride-2 phase decomposition implemented for 1x1/pad0 and 3x3/pad1"
    # Pure device ops with Python-side indices: no index tensor is copied host -> device, so this is legal inside a
    # CUDA-graph capture (the active block's filters are re-packed every step).
    flat = w_krsc.reshape(Co, kh * kw, Ci)
    zero = w_krsc.new_zeros(Co, Ci)
    idx = _tap_index_table(kh).reshape(-1).tolist()
    sel = torch.stack([flat[:, i] if i < kh * kw else zero for i in idx], dim=1).reshape(Co, 2, 2, 2, 2, Ci)   # co ph pw dr ds ci
    return sel.permute(1, 2, 5, 3, 4, 0).reshape(4 * Ci, 2, 2, Co).contiguous()


def dgrad_s2(dy_nhwc: torch.Tensor, w_packed: torch.Tensor, conv2x2: Callable[[torch.Tensor, torch.Tensor], torch.Tensor]
             ) -> torch.Tensor:
    """dy ``[N, Ho, Wo, Co]``, packed filter -> dx ``[N, 2Ho, 2Wo, Ci]``.  ``conv2x2(x, w)`` must return the 2x2,
    stride-1 convolution anchored top-left with zero padding on the bottom/right, output size = input size."""
    N, Ho, Wo, _ = dy_nhwc.shape
    Ci = w_packed.shape[0] // 4
    y = conv2x2(dy_nhwc, w_packed)                                   # [N, Ho, Wo, 4*Ci]  (ph, pw, ci)
    return y.view(N, Ho, Wo, 2, 2, Ci).permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * Ho, 2 * Wo, Ci)


def conv2x2_oracle(x_nhwc: torch.Tensor, w_krsc: torch.Tensor) -> torch.Tensor:
    """ATen oracle of the injected convolution (CPU tests, fall-back)."""
    x = F.pad(x_nhwc.permute(0, 3, 1, 2), (0, 1, 0, 1))
    return F.conv2d(x, w_krsc.permute(0, 3, 1, 2)).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------
# ConvTranspose2d(k=4, stride=2, padding=1) — the VAE decoders (SURVEY G7, /root/reference/src/simple_models.py:262-265,
# :336-340) — as ONE 3x3 / pad 1 / stride 1 convolution with 4*C_out output channels + the same pixel shuffle:
#     y[n, 2i+ph, 2j+pw, co] = sum_{t_r,t_s in {0,1,2}} sum_ci x[n, i+t_r-1, j+t_s-1, ci] * Wp[(ph,pw,co), t_r, t_s, ci]
# phase 0 takes filter rows 3 (offset -1) and 1 (offset 0), phase 1 takes rows 2 (offset 0) and 0 (offset +1); the other
# window position of each phase is zero (4 of 9 taps populated per phase).
# ------------------------------------------------------------------------------------------------
_TAP4 = {(0, 0): 3, (0, 1): 1, (1, 1): 2, (1, 2): 0}      # (phase, window position) -> transposed-filter index


def pack_convT_s2_weight(w_iokk: torch.Tensor) -> torch.Tensor:
    """ConvTranspose2d weight ``[C_in, C_out, 4, 4]`` -> KRSC filter ``[4*C_out, 3, 3, C_in]`` of the equivalent conv."""
    Ci, Co, kh, kw = w_iokk.shape
    assert kh == 4 and kw == 4, "phase decomposition implemented for ConvTranspose2d(k=4, stride=2, padding=1)"
    zero = w_iokk.new_zeros(Co, Ci)
    taps = []
    for ph in (0, 1):
        for pw in (0, 1):
            for tr in (0, 1, 2):
                for ts in (0, 1, 2):
                    r, s_ = _TAP4.get((ph, tr)), _TAP4.get((pw, ts))
                    taps.append(w_iokk[:, :, r, s_].t() if (r is not None and s_ is not None) else zero)   # [Co, Ci]
    sel = torch.stack(taps, dim=0).reshape(2, 2, 3, 3, Co, Ci)                   # ph pw tr ts co ci
    return sel.permute(0, 1, 4, 2, 3, 5).reshape(4 * Co, 3, 3, Ci).contiguous()


def convT_s2(x_nhwc: torch.Tensor, w_packed: torch.Tensor, conv3x3: Callable[[torch.Tensor, torch.Tensor], torch.Tensor]
             ) -> torch.Tensor:
    """x ``[N, H, W, Ci]`` -> ``[N, 2H, 2W, Co]``; ``conv3x3(x, w)`` = 3x3 / pad 1 / stride 1 convolution (bias and
    activation, if any, are applied by the caller's ``conv3x3`` on the 4*Co phase-major channels)."""
    N, H, W, _ = x_nhwc.shape
    Co = w_packed.shape[0] // 4
    y = conv3x3(x_nhwc, w_packed)                                    # [N, H, W, 4*Co]  (ph, pw, co)
    return y.view(N, H, W, 2, 2, Co).permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * H, 2 * W, Co)


def conv3x3_oracle(x_nhwc: torch.Tensor, w_krsc: torch.Tensor) -> torch.Tensor:
    return F.conv2d(x_nhwc.permute(0, 3, 1, 2), w_krsc.permute(0, 3, 1, 2), None, 1, 1).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------
# Multi-dilation convolution (the CPC encoder stem, SURVEY G6, /root/reference/src/simple_models.py:441-460): B convolutions of
# the SAME input with the same k x k / stride, their own dilation d_b / padding p_b and their own output channels, followed by a
# channel concatenation, as ONE implicit GEMM:
#     y[n, ho, wo, (b, co)] = sum_{r, s, ci} x[n, ho*stride + r*d_b - p_b, wo*stride + s*d_b - p_b, ci] * W_b[co, r, s, ci]
# The kernel (csrc/igemm_wgmma.cuh, IgemmParams::ms_*) enumerates "filter rows" R = (b, r) of a merged filter
# Wm[(b', co), (b, r), s, ci] = W_b[co, r, s, ci] if b' == b else 0 (block diagonal), and row R reads the input through branch
# R // k's dilation and padding.  Everything below is plain PyTorch: the packing used by the GPU path and an oracle that gathers
# the taps exactly in the kernel's order.
# ------------------------------------------------------------------------------------------------
def pack_multidil_weight(ws_oikk) -> torch.Tensor:
    """B conv weights ``[Co, Ci, k, k]`` (same shape) -> merged KRSC filter ``[B*Co, B*k, k, Ci]`` (block diagonal)."""
    B = len(ws_oikk)
    Co, Ci, k, _ = ws_oikk[0].shape
    w_all = torch.stack([w.permute(0, 2, 3, 1) for w in ws_oikk])                       # [B, Co, k, k, Ci]
    wm = w_all.new_zeros(B, Co, B, k, k, Ci)
    wm.diagonal(dim1=0, dim2=2).copy_(w_all.permute(1, 2, 3, 4, 0))                     # branch b -> rows (b, :) of its own channels
    return wm.view(B * Co, B * k, k, Ci)


def multidil_conv_oracle(x_nhwc: torch.Tensor, wm: torch.Tensor, k: int, stride: int, dils, pads) -> torch.Tensor:
    """The kernel's tap enumeration in plain PyTorch: for filter row R = (b, r) and column s, one shifted / strided view of the
    zero-padded input times the [C_out_total, C_in] slice of the merged filter."""
    N, H, W, Ci = x_nhwc.shape
    B = len(dils)
    Ho = (H + 2 * pads[0] - dils[0] * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pads[0] - dils[0] * (k - 1) - 1) // stride + 1
    big = max(max(pads), max(d * (k - 1) for d in dils))                                  # enough zero border for every tap
    xp = F.pad(x_nhwc, (0, 0, big, big + stride, big, big + stride))
    y = x_nhwc.new_zeros(N, Ho, Wo, wm.shape[0])
    for R in range(B * k):
        b, r = divmod(R, k)
        d, p = dils[b], pads[b]
        for s in range(k):
            h0, w0 = big + r * d - p, big + s * d - p
            tap = xp[:, h0: h0 + (Ho - 1) * stride + 1: stride, w0: w0 + (Wo - 1) * stride + 1: stride, :]
            y = y + tap @ wm[:, R, s, :].t()
    return y


# ------------------------------------------------------------------------------------------------
# Tap packing (IgemmParams::cw): with C_in <= 16 a 32-wide k-block of the implicit GEMM holds 32 / cw filter taps, each as its own
# cw-channel sub-tile, instead of one tap whose channels are padded to 32 with zeros.  k-block kb, sub-tile j covers tap
# t = kb * (32 / cw) + j (taps past kh*kw contribute zeros); the activation sub-tile holds channels [0, C_in) of that tap and
# zeros above, the weight sub-tile is the cw columns of the [C_out, kh*kw*C_in] filter matrix starting at column t * C_in — when
# C_in < cw those columns run into the NEXT tap's weights, which meet the zero channels of the activation sub-tile.
# ------------------------------------------------------------------------------------------------
def tap_packed_gemm_oracle(x_nhwc: torch.Tensor, w_krsc: torch.Tensor, stride: int, pad: int, cw: int) -> torch.Tensor:
    """conv(x, w) evaluated k-block by k-block exactly as the tap-packed kernel feeds the tensor core."""
    N, H, W, Ci = x_nhwc.shape
    Co, kh, kw, _ = w_krsc.shape
    assert Ci <= cw and 32 % cw == 0
    tpk = 32 // cw
    Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    xp = F.pad(x_nhwc, (0, 0, pad, pad, pad, pad))
    wmat = w_krsc.reshape(Co, kh * kw * Ci)
    wmat = F.pad(wmat, (0, 32))                                                           # reads past the filter give zeros (TMA OOB fill)
    taps = kh * kw
    y = x_nhwc.new_zeros(N * Ho * Wo, Co)
    for kb in range(-(-taps // tpk)):
        a = x_nhwc.new_zeros(N * Ho * Wo, 32)
        bmat = x_nhwc.new_zeros(Co, 32)
        for j in range(tpk):
            t = kb * tpk + j
            if t < taps:
                r, s = divmod(t, kw)
                tap = xp[:, r: r + (Ho - 1) * stride + 1: stride, s: s + (Wo - 1) * stride + 1: stride, :]
                a[:, j * cw: j * cw + Ci] = tap.reshape(-1, Ci)                           # channels >= C_in of the sub-tile stay zero
                bmat[:, j * cw: (j + 1) * cw] = wmat[:, t * Ci: t * Ci + cw]              # may run into the next tap's columns
        y = y + a @ bmat.t()
    return y.view(N, Ho, Wo, Co)


# ------------------------------------------------------------------------------------------------
# Shuffle store (csrc/gemm_wgmma.cu: conv2d_nhwc_shuffle_tf32): the phase-packed stride-1 convolution of `dgrad_s2` does not write
# [N, Ho, Wo, (ph, pw, ci)] and shuffle it afterwards; each 32-row x 32-column epilogue chunk (32 consecutive output pixels of the
# packed convolution = 32 / Wo whole rows, 32 consecutive packed channels = one phase, channels ci0 .. ci0+31) is ONE bulk tensor
# store through a 5-D tensor map over the result viewed as {ci, pw, wo, ph, n*Ho + ho} with box {32, 1, Wo, 1, 32 / Wo} at
# coordinates (ci0, pw, 0, ph, row0 / Wo).  Plain-PyTorch model of exactly that addressing:
# ------------------------------------------------------------------------------------------------
def shuffle_store_oracle(y_packed: torch.Tensor) -> torch.Tensor:
    """``[N, Ho, Wo, 4*Ci]`` (channels (ph, pw, ci)) -> ``[N, 2Ho, 2Wo, Ci]`` by 32 x 32 chunk stores with the kernel's coordinates."""
    N, Ho, Wo, C4 = y_packed.shape
    Ci = C4 // 4
    assert Ci % 32 == 0 and 32 % Wo == 0, "a chunk must stay inside one phase and cover whole output rows"
    out = y_packed.new_zeros(N, 2 * Ho, 2 * Wo, Ci)
    view5 = out.view(N * Ho, 2, Wo, 2, Ci)                    # [n*Ho + ho, ph, wo, pw, ci]: the tensor map's dims, slowest first
    rows = y_packed.reshape(N * Ho * Wo, C4)
    for row0 in range(0, rows.shape[0], 32):
        for pc in range(0, C4, 32):
            phase, ci0 = divmod(pc, Ci)
            ph, pw = phase >> 1, phase & 1
            hon0 = row0 // Wo
            nrow = min(32, rows.shape[0] - row0)               # the last chunk is clipped by the tensor map's bounds
            chunk = rows[row0: row0 + nrow, pc: pc + 32].reshape(nrow // Wo, Wo, 32)
            view5[hon0: hon0 + nrow // Wo, ph, :, pw, ci0: ci0 + 32] = chunk
    return out


# ------------------------------------------------------------------------------------------------
# Window reuse (csrc/igemm_wgmma.cuh: igemm_wgmma_pix_kernel with WIN_KH > 0): for a stride-1, dilation-1 convolution a
# 256-pixel tile of `rows` whole output rows of one image (first row h0) is
#     y_tile = sum_{s, cb} sum_{r < kh} window_{s,cb}[r : r + rows] @ W[:, r, s, cb * 32 : cb * 32 + 32]^T
# where window_{s,cb} is ONE box of rows + kh - 1 input rows starting at h0 - pad, columns shifted by s - pad and channels
# [cb * 32, cb * 32 + 32), zero outside the image (the TMA zero fill): filter row r reads the same box from row r on.
# ------------------------------------------------------------------------------------------------
def window_reuse_conv_oracle(x_nhwc: torch.Tensor, w_krsc: torch.Tensor, pad: int, rows: int) -> torch.Tensor:
    """Stride-1 convolution of ``x [N, H, W, Ci]`` with ``w [Co, kh, kw, Ci]`` evaluated tile by tile and window by window
    exactly as the window-reuse kernel accumulates it; ``rows`` output rows per tile (must divide H_out)."""
    N, H, W, Ci = x_nhwc.shape
    Co, kh, kw, _ = w_krsc.shape
    Ho, Wo = H + 2 * pad - kh + 1, W + 2 * pad - kw + 1
    assert Ho % rows == 0, "a tile is whole output rows of one image"
    win_rows = rows + kh - 1
    y = x_nhwc.new_zeros(N, Ho, Wo, Co)
    for n in range(N):
        for h0 in range(0, Ho, rows):
            acc = x_nhwc.new_zeros(rows * Wo, Co)
            for s in range(kw):
                for c0 in range(0, Ci, 32):
                    c1 = min(c0 + 32, Ci)
                    window = x_nhwc.new_zeros(win_rows, Wo, c1 - c0)           # out-of-image rows / columns stay zero
                    for i in range(win_rows):
                        hi = h0 - pad + i
                        if not 0 <= hi < H:
                            continue
                        w_lo, w_hi = max(0, s - pad), min(W, s - pad + Wo)       # input columns inside the image
                        if w_lo < w_hi:
                            window[i, w_lo - (s - pad): w_hi - (s - pad)] = x_nhwc[n, hi, w_lo:w_hi, c0:c1]
                    for r in range(kh):
                        acc = acc + window[r: r + rows].reshape(rows * Wo, c1 - c0) @ w_krsc[:, r, s, c0:c1].t()
            y[n, h0: h0 + rows] = acc.view(rows, Wo, Co)
    return y
