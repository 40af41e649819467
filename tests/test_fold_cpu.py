"""The fold of the last upsampler with R-CNN1 (engine.cu build_fold / fold_dot, train.cuh fold_kernel), the parts that
need no GPU.

At inference the last depth_to_space layer (Up-PS, Up-PS2 at x4, or Up-TCNN in its 3x3 LR form) and a 3x3 R-CNN1 are
both linear, so the engine packs the layer
    W'[tap][ci][ij*9 + t] = sum_c W[tap][ci][ij*C + c] w_r[t][c],   b'[ij*9 + t] = sum_c b[ij*C + c] w_r[t][c]
stores its column (ij, t) at LR pixel (y, x) into tap plane t at HR pixel (s*y + i, s*x + j) (EPI_D2S_TAPS), and
conv_last_gather adds tap t of the HR pixel shifted by (t / 3 - 1, t % 3 - 1) where that pixel lies inside the image.
Here that chain, restated in numpy, is held against the oracle's upsampler -> depth_to_space -> R-CNN1 in fp64, on
images one pixel tall, one pixel wide and of odd sizes, so that every border case of the gather is reached.  The fp32
rounding of the fold is pinned too: exact products summed in fp64 in ascending c, one rounding, whether or not the
compiler contracts the sum into fused multiply-adds."""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcscn_oracle as O
import tconv_oracle as T


def conv(a, w_hwio):
    """tf.nn.conv2d(SAME) in fp64 of an NCHW array with an HWIO filter."""
    w = torch.from_numpy(np.ascontiguousarray(w_hwio, np.float64)).permute(3, 2, 0, 1)
    return F.conv2d(torch.from_numpy(np.ascontiguousarray(a, np.float64)), w, padding=w.shape[-1] // 2).numpy()


def fold64(w, b, wr, c):
    """W' and b' in fp64: w [k, k, cin, sub*C], b [sub*C], wr [3, 3, C, 1]."""
    k, _, cin, cols = w.shape
    sub = cols // c
    r = wr.reshape(9, c).astype(np.float64)
    wf = np.einsum("yxisc,tc->yxist", w.astype(np.float64).reshape(k, k, cin, sub, c), r).reshape(k, k, cin, sub * 9)
    bf = np.einsum("sc,tc->st", b.astype(np.float64).reshape(sub, c), r).reshape(sub * 9)
    return wf, bf


def fold_dot(a, w):
    """engine.cu fold_dot: sum over c of fp64(a[c]) * fp64(w[c]), c ascending, each add rounded to fp64."""
    s = 0.0
    for x, y in zip(a.tolist(), w.tolist()):
        s += x * y
    return s


def fold_dot_fma(a, w):
    """The same sum with every step a fused multiply-add, round(s + a*b) once, computed exactly with fractions."""
    s = 0.0
    for x, y in zip(a.tolist(), w.tolist()):
        s = float(Fraction(s) + Fraction(x) * Fraction(y))
    return s


def fold32(w, b, wr, c, dot=fold_dot):
    """W' and b' as build_fold / fold_kernel form them: fp32 inputs, fold_dot, one rounding to fp32."""
    k, _, cin, cols = w.shape
    sub = cols // c
    r = wr.reshape(9, c)
    rows = w.reshape(k * k * cin, sub, c)
    wf = np.array([[[dot(rows[q, ij], r[t]) for t in range(9)] for ij in range(sub)] for q in range(rows.shape[0])])
    bf = np.array([[dot(b.reshape(sub, c)[ij], r[t]) for t in range(9)] for ij in range(sub)])
    return wf.astype(np.float32).reshape(k, k, cin, sub * 9), bf.astype(np.float32).reshape(sub * 9)


def taps_and_gather(a, wf, bf, s):
    """The folded layer at LR, the EPI_D2S_TAPS store into tap planes [9][n][sH][sW], and conv_last_gather."""
    out = conv(a, wf) + bf.reshape(1, -1, 1, 1)                      # [n, s*s*9, H, W]
    n, _, h, w = out.shape
    v = out.reshape(n, s, s, 9, h, w).transpose(3, 0, 4, 1, 5, 2).reshape(9, n, s * h, s * w)
    y = np.zeros((n, s * h, s * w))
    for t in range(9):
        dy, dx = t // 3 - 1, t % 3 - 1
        p = np.pad(v[t], ((0, 0), (1, 1), (1, 1)))                   # taps outside the image add nothing
        y += p[:, 1 + dy:1 + dy + s * h, 1 + dx:1 + dx + s * w]
    return y


def chain(a, w, b, wr, s):
    """The oracle's order: upsampler, depth_to_space(s), R-CNN1 (fp64)."""
    up = O.depth_to_space(torch.from_numpy(conv(a, w) + b.reshape(1, -1, 1, 1)), s)
    return O.conv2d_same(up, wr, torch.float64).numpy()[:, 0]


SHAPES = [(1, 1, 1), (1, 1, 5), (1, 4, 1), (2, 3, 5)]
C = 16


def weights(k, cin, sub, seed):
    g = np.random.RandomState(seed)
    w = (g.randn(k, k, cin, sub * C) * 0.2).astype(np.float32)
    b = (g.randn(sub * C) * 0.1).astype(np.float32)
    wr = (g.randn(3, 3, C, 1) * 0.3).astype(np.float32)
    return w, b, wr


@pytest.mark.parametrize("s,cin", [(2, 24), (3, 24), (2, 16), (8, 24)], ids=["Up-PS-x2", "Up-PS-x3", "Up-PS2-x4", "Up-PS-x8"])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % sh for sh in SHAPES])
def test_pixel_shuffler_fold_equals_chain(s, cin, shape):
    """Up-PS at x2, x3, x8 and the x2 Up-PS2 stage of x4 (its input is the first stage's C channels)."""
    w, b, wr = weights(3, cin, s * s, seed=s + cin)
    a = np.random.RandomState(1).rand(shape[0], cin, shape[1], shape[2]) * 4 - 1
    ref = chain(a, w, b, wr, s)
    wf, bf = fold64(w, b, wr, C)
    got = taps_and_gather(a, wf, bf, s)
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("s", [2, 4, 8])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % sh for sh in SHAPES])
def test_transposed_upsampler_fold_equals_chain(s, shape):
    """Up-TCNN: the fold of its 3x3 LR filter (structural zeros included) against conv2d_transpose -> R-CNN1, which
    has no depth_to_space step of its own; no bias."""
    g = np.random.RandomState(10 + s)
    tw = (g.randn(T.ksize(s), T.ksize(s), C, C) * 0.2).astype(np.float32)
    wr = (g.randn(3, 3, C, 1) * 0.3).astype(np.float32)
    a = np.random.RandomState(2).rand(shape[0], C, shape[1], shape[2]) * 4 - 1
    up = T.conv_transpose(torch.from_numpy(a), tw.astype(np.float64), s)
    ref = O.conv2d_same(up, wr, torch.float64).numpy()[:, 0]
    wf, bf = fold64(T.tconv_filter(tw, s), np.zeros(s * s * C, np.float32), wr, C)
    got = taps_and_gather(a, wf, bf, s)
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_fp32_fold_is_one_rounding_with_or_without_fma():
    """fp32 products are exact in fp64 (48 significant bits), so a fused multiply-add rounds each step exactly as a
    separate add does: the host fold and the device fold_kernel agree whatever either compiler contracts.  The result is
    the fp64 sum rounded once to fp32."""
    w, b, wr = weights(3, 3, 4, seed=7)
    for x, y in zip(w.ravel()[:64].tolist(), wr.ravel()[:64].tolist()):
        assert Fraction(x) * Fraction(y) == Fraction(x * y)
    wf, bf = fold32(w, b, wr, C)
    wf_fma, bf_fma = fold32(w, b, wr, C, dot=fold_dot_fma)
    assert np.array_equal(wf.view(np.uint32), wf_fma.view(np.uint32))
    assert np.array_equal(bf.view(np.uint32), bf_fma.view(np.uint32))
    w64, b64 = fold64(w, b, wr, C)
    assert np.all(np.abs(wf - w64) <= 2.0 ** -24 * (1 + 1e-9) * np.abs(w64) + 1e-45)
    assert np.all(np.abs(bf - b64) <= 2.0 ** -24 * (1 + 1e-9) * np.abs(b64) + 1e-45)
