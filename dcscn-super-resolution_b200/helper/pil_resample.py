"""
Bit-exact restatement of Pillow's bicubic `Image.resize` for single-channel float images (mode 'F'), the resampler behind
`util.resize_image_by_pil` (reference helper/utilty.py:211-239) that produces the network's second input `x2` and the
low-resolution input itself.

Pillow (src/libImaging/Resample.c) resizes in two passes - horizontal, then vertical - and for mode 'F':
  * per output coordinate it precomputes a window [xmin, xmin + n) and double-precision weights
    w(x) = bicubic((x + xmin - center + 0.5) / filterscale), a = -0.5, normalised by their sum, with
    center = (xx + 0.5) * in/out, filterscale = max(in/out, 1), support = 2 * filterscale;
  * every output sample is  (float) sum_x (double)pixel * w(x)  accumulated in a double, in window order; the
    intermediate image between the two passes is float32.
`precompute_coeffs` below builds exactly those tables; `resize_float` applies them with numpy in the same operation order
(tests/test_host.py holds it bit for bit to Pillow), and the CUDA kernels of csrc/conv_aux.cuh (`pil_resample_*`) apply the
same tables on the device with non-fused double multiplies / adds - so `x2` can be formed in HBM from the LR image alone.
"""

import math

import numpy as np


def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def precompute_coeffs(in_size, out_size):
    """(weights float64 [out_size, ksize], bounds int32 [out_size, 2] = (first input index, taps)) of one axis."""
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    kk = np.zeros((out_size, ksize), dtype=np.float64)
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        ww = 0.0
        for x in range(xmax):
            w = _bicubic((x + xmin - center + 0.5) * ss)
            kk[xx, x] = w
            ww += w
        if ww != 0.0:
            for x in range(xmax):
                kk[xx, x] /= ww
        bounds[xx] = (xmin, xmax)
    return kk, bounds


def resize_float(image, out_width, out_height):
    """Pillow's `Image.fromarray(image).resize([out_width, out_height], Image.BICUBIC)` for a 2-D float array."""
    img = np.asarray(image, dtype=np.float32)
    h, w = img.shape
    kx, bx = precompute_coeffs(w, out_width)
    ky, by = precompute_coeffs(h, out_height)
    tmp = np.empty((h, out_width), dtype=np.float32)
    for xx in range(out_width):
        x0, n = bx[xx]
        acc = np.zeros(h, dtype=np.float64)
        for x in range(n):
            acc = acc + img[:, x0 + x].astype(np.float64) * kx[xx, x]
        tmp[:, xx] = acc.astype(np.float32)
    out = np.empty((out_height, out_width), dtype=np.float32)
    for yy in range(out_height):
        y0, n = by[yy]
        acc = np.zeros(out_width, dtype=np.float64)
        for y in range(n):
            acc = acc + tmp[y0 + y, :].astype(np.float64) * ky[yy, y]
        out[yy, :] = acc.astype(np.float32)
    return out


def _coeffs_8bpc(kk):
    """Pillow's normalize_coeffs_8bpc: the double weights as 22-bit fixed point, rounded half away from zero."""
    scaled = kk * (1 << 22)
    return np.where(kk < 0, np.trunc(scaled - 0.5), np.trunc(scaled + 0.5)).astype(np.int64)


def _clip8(ss):
    return np.clip(ss >> 22, 0, 255).astype(np.uint8)


def resize_uint8(image, out_width, out_height):
    """Pillow's `Image.fromarray(image).resize([out_width, out_height], Image.BICUBIC)` for a 2-D uint8 array (mode 'L',
    ImagingResampleHorizontal_8bpc / ImagingResampleVertical_8bpc): the same tables as `resize_float` in 22-bit fixed
    point, an int32 sum that starts at 2^21, clamp(sum >> 22, 0, 255), and a uint8 image between the two passes.  The
    device kernels `pil_resample8_h/v_kernel` (csrc/conv_aux.cuh) apply it to the mode-'L' crops of a mini-batch."""
    img = np.asarray(image, dtype=np.uint8).astype(np.int64)
    h, w = img.shape
    kx, bx = precompute_coeffs(w, out_width)
    ky, by = precompute_coeffs(h, out_height)
    kx, ky = _coeffs_8bpc(kx), _coeffs_8bpc(ky)
    tmp = np.empty((h, out_width), dtype=np.int64)
    for xx in range(out_width):
        x0, n = bx[xx]
        tmp[:, xx] = _clip8((1 << 21) + img[:, x0:x0 + n] @ kx[xx, :n])
    out = np.empty((out_height, out_width), dtype=np.uint8)
    for yy in range(out_height):
        y0, n = by[yy]
        out[yy, :] = _clip8((1 << 21) + ky[yy, :n] @ tmp[y0:y0 + n, :])
    return out
