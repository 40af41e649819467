"""The fp64 oracle (oracle/dcscn_oracle.py) for --pixel_shuffler=false: the upsampler is Up-TCNN, one
tf.nn.conv2d_transpose(stride s, SAME) with the variable Up-TCNN/Tconv_W [K, K, C, C] (TF's [h, w, out, in] layout,
K = 2s - s%2), no bias and no activation, in place of Up-PS [+ Up-PS2] (helper/tf_graph.py:219-236, called at
DCSCN.py:310-311).  C = nin_filters + nin_filters2, and R-CNN1 reads those C channels (pixel_shuffler_filters is
ignored on this path).  Under --depthwise_separable the other layers are separable and Up-TCNN stays dense.

Besides the torch form (F.conv_transpose2d) this module states the layer two more ways, for the tests that pin the
engine's sub-pixel form of it:
  * `scatter_reference`: a literal loop over TF's definition, out[i*s + k - pad_top] += in[i] * W[k], per axis;
  * `tconv_filter` / `gather_conv`: the 3x3 LR filter F the engine packs (engine.cu tconv_filter_map), then the DCR
    depth_to_space(s) of the oracle."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import dcscn_oracle as O

TCONV = "Up-TCNN/Tconv_W"


def ksize(s):
    return 2 * s - s % 2                                   # util.get_upscale_filter_size


def pad_top(s):
    return (ksize(s) - s) // 2                             # SAME: pad_total = K - s for an output of s * H


class Config(O.OracleConfig):
    """OracleConfig with the flag; `transposed_upsampler=True` is --pixel_shuffler=false."""

    def __init__(self, transposed_upsampler=True, **kw):
        super().__init__(**kw)
        self.transposed_upsampler = transposed_upsampler


def upsampler_channels(cfg):
    return cfg.nin_filters + cfg.nin_filters2


def layer_table(cfg):
    """dcscn_oracle.layer_table with the pixel-shuffler entries replaced by ("Up-TCNN", K, C, C, False, False)."""
    table = [e for e in O.layer_table(cfg) if not e[0].startswith("Up-PS")]
    c = upsampler_channels(cfg)
    i = [e[0] for e in table].index("B2") + 1
    table.insert(i, ("Up-TCNN", ksize(cfg.scale), c, c, False, False))
    # R-CNN1 reads the C channels of the transposed convolution
    return [(sc, k, c, co, b, p) if sc == "R-CNN1" else (sc, k, ci, co, b, p) for sc, k, ci, co, b, p in table]


def variable_names(cfg):
    names = []
    for scope, k, cin, cout, bias, prelu in layer_table(cfg):
        if scope == "Up-TCNN":
            names.append(TCONV)
            continue
        names.append(scope + "/conv_W")
        if bias:
            names.append(scope + "/conv_B")
        if cfg.depthwise_separable:
            names.append(scope + "/depthwise_W")
            names.append(scope + "/pointwise_W")
        if prelu:
            names.append("%s/prelu/%s_prelu" % (scope, scope.split("/")[-1]))
    return names


def random_weights(cfg, seed=0):
    """He-style weights for every layer (dcscn_oracle.he_init_weights) and a random Tconv_W with the scale of the
    bilinear initial value (entries up to 1, summing to about s*s per output pixel and channel): random so that every
    tap and every channel pair carries its own value."""
    w = O.he_init_weights(cfg, seed=seed)           # draws the pixel-shuffler filters too; they are dropped below
    c = upsampler_channels(cfg)
    k = ksize(cfg.scale)
    g = np.random.RandomState(seed + 101)
    tw = g.randn(k, k, c, c) * (cfg.scale / (k * math.sqrt(c)))
    for i in range(c):
        tw[:, :, i, i] += bilinear(k)
    w[TCONV] = tw.astype(np.float32)
    # R-CNN1 has C inputs here (pixel_shuffler_filters does not apply)
    r = g.randn(cfg.cnn_size, cfg.cnn_size, c, 1) * math.sqrt(2.0 / (cfg.cnn_size ** 2 * c))
    w["R-CNN1/conv_W"] = np.clip(r, -2, 2).astype(np.float32)
    if cfg.depthwise_separable:
        w["R-CNN1/depthwise_W"] = (g.randn(cfg.cnn_size, cfg.cnn_size, c, 1) * 0.2 + 1.0 / cfg.cnn_size ** 2).astype(np.float32)
        w["R-CNN1/pointwise_W"] = (g.randn(1, 1, c, 1) * math.sqrt(2.0 / c)).astype(np.float32)
    return {n: w[n] for n in variable_names(cfg)}


def bilinear(size):
    """utilty.upsample_filter restated: the separable tent of half-width ceil(size / 2) around the kernel centre."""
    factor = (size + 1) // 2
    center = factor - 1 if size % 2 == 1 else factor - 0.5
    t = 1 - np.abs(np.arange(size) - center) / factor
    return np.outer(t, t)


def conv_transpose(x_nchw, w_kkoi, s):
    """tf.nn.conv2d_transpose(stride s, SAME) to an s x larger output: K - s is even at s = 2, 3, 4, so torch's
    symmetric padding (K - s) / 2 gives exactly TF's output of s*H x s*W."""
    w = w_kkoi if torch.is_tensor(w_kkoi) else torch.from_numpy(np.ascontiguousarray(w_kkoi)).to(x_nchw.dtype)
    return F.conv_transpose2d(x_nchw, w.permute(3, 2, 0, 1), stride=s, padding=pad_top(s))


def scatter_reference(x_nchw, w_kkoi, s):
    """TF's definition as a literal loop (fp64 numpy): out[o] += in[i] W[k] for o = i*s + k - pad_top, per axis."""
    x = np.asarray(x_nchw, np.float64)
    w = np.asarray(w_kkoi, np.float64)
    n, c, h, wd = x.shape
    k, pt = ksize(s), pad_top(s)
    out = np.zeros((n, w.shape[2], s * h, s * wd))
    for i in range(h):
        for j in range(wd):
            for ky in range(k):
                oy = i * s + ky - pt
                if oy < 0 or oy >= s * h:
                    continue
                for kx in range(k):
                    ox = j * s + kx - pt
                    if 0 <= ox < s * wd:
                        out[:, :, oy, ox] += x[:, :, i, j] @ w[ky, kx].T     # [n, ci] x [ci, co]
    return out


def tconv_filter_index(s, c):
    """Index into Tconv_W.ravel() of every entry of the 3x3 LR filter F [3, 3, C, s*s*C] (HWIO), -1 where F is a
    structural zero: F[dy+1][dx+1][ci][(py*s + px)*C + co] = W[py + pad_top - s*dy][px + pad_top - s*dx][co][ci]."""
    k, pt = ksize(s), pad_top(s)
    idx = -np.ones((3, 3, c, s * s * c), np.int64)
    flat = np.arange(k * k * c * c).reshape(k, k, c, c)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            for py in range(s):
                for px in range(s):
                    ky, kx = py + pt - s * dy, px + pt - s * dx
                    if 0 <= ky < k and 0 <= kx < k:
                        col = (py * s + px) * c
                        idx[dy + 1, dx + 1, :, col:col + c] = flat[ky, kx].T     # [ci, co]
    return idx


def tconv_filter(w_kkoi, s):
    c = w_kkoi.shape[2]
    idx = tconv_filter_index(s, c)
    f = np.where(idx >= 0, np.asarray(w_kkoi).ravel()[np.maximum(idx, 0)], 0)
    return f.astype(np.asarray(w_kkoi).dtype)


def tconv_filter_grad(df, s, c):
    """The inverse gather: dW from the gradient of F."""
    idx = tconv_filter_index(s, c)
    k = ksize(s)
    dw = np.zeros(k * k * c * c, df.dtype)
    m = idx >= 0
    dw[idx[m]] = df[m]
    return dw.reshape(k, k, c, c)


def gather_conv(x_nchw, w_kkoi, s):
    """The engine's form: a 3x3 SAME convolution with F, then depth_to_space(s)."""
    f = torch.from_numpy(tconv_filter(np.asarray(w_kkoi, np.float64), s))
    return O.depth_to_space(F.conv2d(torch.as_tensor(x_nchw, dtype=torch.float64), f.permute(3, 2, 0, 1), padding=1), s)


class Oracle(O.Oracle):
    """dcscn_oracle.Oracle with Up-TCNN as the upsampler, forward and autograd train step."""

    def __init__(self, cfg, weights, dtype=torch.float64):
        super().__init__(cfg, weights, dtype)
        self.table = layer_table(cfg)

    def forward_nchw(self, x, x2, params=None, keep_prob=1.0, masks=None, return_intermediates=False):
        cfg = self.cfg
        p = params if params is not None else self.w
        inter = {}
        feats = []
        h = x
        for i in range(cfg.layers):
            h = self._layer("CNN%d" % (i + 1), h, params, keep_prob, masks)
            feats.append(h)
            inter["CNN%d" % (i + 1)] = h
        hc = torch.cat(feats, dim=1)
        a1 = self._layer("A1", hc, params, keep_prob, masks)
        b1 = self._layer("B1", hc, params, keep_prob, masks)
        b2 = self._layer("B2", b1, params, keep_prob, masks)
        inter["A1"], inter["B1"], inter["B2"] = a1, b1, b2
        h = torch.cat([b2, a1], dim=1)
        tw = p[TCONV] if torch.is_tensor(p[TCONV]) else O._t(p[TCONV], self.dtype)
        h = conv_transpose(h, tw, cfg.scale)
        inter["Up-TCNN"] = h
        h = self._layer("R-CNN1", h, params)
        inter["R-CNN"] = h
        y = h + x2
        if return_intermediates:
            return y, inter
        return y

    def trainable_names(self):
        return variable_names(self.cfg)

    def l2_weight_names(self):
        return [TCONV if scope == "Up-TCNN" else scope + "/conv_W" for scope, *_ in self.table]
