"""
Forward parity of every kernel and layout the inference planner can select (engine.cu: make_tc / choose_tiling,
choose_patch, get_plan's fused_last / rdot_parts, issue_front, forward_impl, forward_ds_tile), at both operand
precisions.  Each case records its first forward with torch.profiler and asserts the kernels it reached, so a change
to a selection rule cannot quietly move a case onto another path.  A CPU test checks that every inference kernel the
library contains is named by some case here.

Tensor-core graphs are held to two references:
  * end to end (f16x3): the fp64 oracle with the stress bars of test_gpu_forward.py, and the CUDA-core cross-check;
  * isolated per layer (f16x3 and f16x1): every layer recomputed in fp64 from the input the GPU itself stored
    (get_activation: the exact fp16 value in f16x1, hi + lo in f16x3), with its weights quantised as pack_tc_layer does
    (one power-of-two scale s per packed layer; fp16(fp32(w) s), plus fp16(fp32(w s) - hi) in f16x3).  No error comes
    in from earlier layers, so the bar follows from the arithmetic of the one kernel, per output element, with
    S = sum |a| |w| of its products:
      output rounding   f16x1: one fp16 ulp of the reference value; f16x3: the hi / lo split, 2^-22 |v| + 2^-25;
                        none for fp32 outputs (Up-PS through EPI_D2S_F32, R-CNN1 + x2 up to its final add, 2^-24 |y|)
      a_lo * w_lo       f16x3 drops it: at most 2^-22 S
      tensor cores      the dom chain of a promotion segment (at most 4 seg_chunks k16 steps) truncates once per step,
                        and each segment is promoted with two round-to-nearest adds: (chain + segments) 2^-23 S
                        (conv_tc.cuh; the correction chain's truncations are 2^-10 of that, counted as one more step)
      fp32 CUDA cores   CNN1, R-CNN1 and the fused R-CNN1 gather: k^2 C 2^-24 S
      epilogue          scale + bias and the PReLU product, each rounded once: 2^-23 (S + |bias|)
      activation        relu / leaky_relu as PReLU; sigmoid, tanh, selu: act_curve's libdevice error (CURVE_U) and the
                        bar of z carried through max |f'| (activation); the train step's dropout: 2^-24 more, dropped
                        elements exactly 0
The fused R-CNN1 output is checked against R-CNN1(Up-PS_ref) + x2, where Up-PS_ref is the last pixel-shuffler layer
computed from the GPU's own input to it; its accumulation bar is carried through |R-CNN1 filter|.

Depthwise-separable graphs (fp32 CUDA cores) are held to the bars of check_depthwise_separable_layers.
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcscn_oracle as O
from conftest import PKG
from test_gpu_forward import SMALL, TOL, assert_stress, gpu_forward, make_engine
from test_gpu_train import DS3, DS4W, assert_kernels_ran, launched_kernels

U23, U24 = 2.0 ** -23, 2.0 ** -24


def pad16(v):
    return (v + 15) // 16 * 16


def tc(*widths):
    """conv_tc_kernel instantiations; {P} becomes the operand plane count of the precision under test."""
    return ["conv_tc_kernel<{P}, %d>" % n for n in widths]


FIRST3 = "conv_first3x3_kernel<false>"

# Tensor-core cases: He-init SMALL with the keys shown changed.  The patch choose_patch picks for a 3 x 3 layer (1 x 1
# layers take the same unless noted): 9 x 11 images take 8 x 16; 2 x 130 take 2 x 64; 1 x 200 take 1 x 128 in f16x1,
# and in f16x3 1 x 128 for 1 x 1 layers and for B2 (16 columns: its weight tiles are small enough for the 128-pixel-wide
# box) but 2 x 64 for the wider 3 x 3 layers; 128 x 1 takes 128 x 1 for 1 x 1 layers and 16 x 8 for 3 x 3 ones.  The
# x4 Up-PS2 runs at twice the LR size: 18 x 22 pixels take 4 x 32, 14 x 66 (a 7 x 33 image) take 16 x 8.  5 x 5 layers
# choose the same way.
X2R = dict(SMALL, nin_filters=16, nin_filters2=16)
TC_CASES = [
    # id, config, (n, h, w), kernels that must run
    # Up-PS 128 columns as 2 x 64, fused R-CNN1 with one partial-plane set; HR width 22: one-pixel gather
    ("x2-rdot1", X2R, (1, 9, 11), [FIRST3] + tc(16, 32, 64) + ["conv_last_gather_kernel"]),
    # 2 x 64 patches; HR width 260: four-pixel gather
    ("x2-rdot1-2x130", X2R, (2, 2, 130), [FIRST3] + tc(16, 32, 64) + ["conv_last_gather4_kernel"]),
    # Up-PS 288 columns as 5 tiles of 64, the last half padding, fused
    ("x3-rdot1", dict(X2R, scale=3), (1, 9, 11), [FIRST3] + tc(16, 32, 64) + ["conv_last_gather_kernel"]),
    ("x3-rdot1-1x200", dict(X2R, scale=3), (1, 1, 200), [FIRST3] + tc(16, 32, 64) + ["conv_last_gather4_kernel"]),
    # fused on Up-PS2 with one partial-plane set; Up-PS through the vector EPI_D2S_PLANES store
    ("x4-rdot1", dict(X2R, scale=4), (1, 7, 33), [FIRST3] + tc(16, 32, 64) + ["conv_last_gather4_kernel"]),
    # Up-PS 192 columns as 2 x 96, fused
    ("x2-ps48", dict(SMALL, nin_filters=32, nin_filters2=16), (1, 9, 11),
     [FIRST3] + tc(16, 32, 48, 96) + ["conv_last_gather_kernel"]),
    # 20 pixel-shuffler channels: element-wise EPI_D2S_PLANES (split_f16) and EPI_D2S_F32, R-CNN1 C = 20
    ("x4-c20", dict(SMALL, scale=4, nin_filters=12, nin_filters2=8), (1, 9, 11),
     [FIRST3] + tc(16, 32, 80) + ["conv_last_kernel"]),
    # 1 x 1 CNN1 (general kernel), CNN / Up-PS layers and R-CNN1
    ("k1-x3", dict(SMALL, scale=3, cnn_size=1), (1, 9, 11), ["conv_first_kernel"] + tc(16, 32, 48, 96) + ["conv_last_kernel"]),
    ("k1-x3-128x1", dict(SMALL, scale=3, cnn_size=1), (1, 128, 1),
     ["conv_first_kernel"] + tc(16, 32, 48, 96) + ["conv_last_kernel"]),
    # 5 x 5 Up-PS / Up-PS2, vector EPI_D2S_F32, R-CNN1 k = 5 with C = 32
    ("k5-x4", dict(X2R, scale=4, cnn_size=5), (1, 7, 33), ["conv_first_kernel"] + tc(16, 32, 64) + ["conv_last_kernel"]),
    # CNN1 with 272 filters (n_pad > 256) on the general kernel; CNN2 ends on a 16-channel K chunk (272 = 4 x 64 + 16)
    ("cnn1-272", dict(SMALL, layers=2, filters=272, min_filters=32), (1, 9, 11),
     ["conv_first_kernel"] + tc(16, 32, 48, 80) + ["conv_last_kernel"]),
    # Up-PS 512 columns as 5 x 112 (7 column chunks per tile: not fusable), R-CNN1 C = 128
    ("ps128", dict(SMALL, nin_filters=96, nin_filters2=32), (1, 9, 11), [FIRST3] + tc(32, 64, 112) + ["conv_last_kernel"]),
    # 576 columns as 6 x 96, unfused (C = 144 > 128)
    ("ps144", dict(SMALL, nin_filters=96, nin_filters2=48), (1, 9, 11),
     [FIRST3] + tc(32, 48, 80, 96) + ["conv_last_kernel"]),
    # 9-column Up-PS in one 16-column tile, element-wise EPI_D2S_F32, R-CNN1 C = 1
    ("x3-ps1", dict(SMALL, scale=3, pixel_shuffler_filters=1), (1, 9, 11), [FIRST3] + tc(16, 32, 48) + ["conv_last_kernel"]),
]

# Depthwise-separable cases (ds_tile_kernel<k, columns / 4>: the column count is the layer's output channels rounded up
# to 4, capped at 32).
DSK1 = dict(scale=3, layers=4, filters=32, min_filters=8, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
            pixel_shuffler_filters=1, depthwise_separable=True, cnn_size=1)     # CNN 32, 20, 13, 8 channels
DSN4 = dict(scale=2, layers=3, filters=28, min_filters=20, filters_decay_gamma=1.5, nin_filters=2, nin_filters2=2,
            pixel_shuffler_filters=1, depthwise_separable=True)                 # CNN 28, 22, 20; A1 | B1 4 columns
DS_CASES = [
    # HR width 27: the one-pixel 3 x 3 R-CNN1
    ("ds-x3-oddw", DS3, (2, 7, 9), ["ds_tile_kernel<3, 4>", "ds_tile_kernel<3, 2>", "ds_tile_kernel<1, 4>",
                                    "ds_single_kernel<3>"]),
    # R-CNN1 12 -> 1 through ds_tile_kernel with `add`; 48-column Up-PS / Up-PS2 on the depthwise cache
    ("ds-x4-wide", DS4W, (2, 6, 5), ["ds_tile_kernel<3, 8>", "ds_tile_kernel<3, 1>", "ds_tile_kernel<3, 2>"]),
    # 1 x 1 CNN and Up-PS layers; 1 x 1 R-CNN1 on the one-pixel kernel
    ("ds-k1-x3", DSK1, (2, 7, 9), ["ds_tile_kernel<1, 8>", "ds_tile_kernel<1, 6>", "ds_tile_kernel<1, 4>",
                                   "ds_tile_kernel<1, 2>", "ds_tile_kernel<3, 2>", "ds_single_kernel<1>"]),
    # A1 | B1 with 4 columns; HR width 20: the four-pixel R-CNN1
    ("ds-nin4-x2", DSN4, (2, 9, 10), ["ds_tile_kernel<3, 8>", "ds_tile_kernel<3, 6>", "ds_tile_kernel<1, 1>",
                                      "ds_tile_kernel<3, 1>", "ds_single4_kernel"]),
]


# ------------------------------------------------------------------------------------ isolated per-layer reference ----
def nchw(a, device=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(device).permute(0, 3, 1, 2)


def conv(a, w):
    """tf.nn.conv2d(SAME) of an NCHW fp64 tensor with an HWIO filter, on the tensor's device."""
    w = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float64)).to(a.device).permute(3, 2, 0, 1)
    return F.conv2d(a, w, padding=w.shape[-1] // 2)


def col(v, device=None):
    """A per-channel vector as an fp64 [1, C, 1, 1] tensor."""
    return torch.from_numpy(np.asarray(v, dtype=np.float64)).to(device).view(1, -1, 1, 1)


def quantise(ws, npl):
    """The operand values pack_tc_layer gives the tensor cores for the weight arrays of one packed layer, over its
    power-of-two scale: s = 2^floor(log2(16384 / max|w|)), hi = fp16(fp32(w) s), lo = fp16(fp32(w s) - hi) (f16x3)."""
    maxw = max(float(np.abs(w).max()) for w in ws)
    s = 2.0 ** np.floor(np.log2(16384.0 / maxw)) if maxw > 0 else 1.0
    out = []
    for w in ws:
        v = w.astype(np.float32) * np.float32(s)
        hi = v.astype(np.float16)
        q = hi.astype(np.float64)
        if npl == 2:
            q = q + (v - hi.astype(np.float32)).astype(np.float16).astype(np.float64)
        out.append(q / s)
    return out


def tc_units(k, cin_pad, seg, npl):
    """Accumulation bar of a tensor-core layer in units of 2^-23 S: (chain + segments), plus the dropped a_lo w_lo
    product (2) and the correction chain (1) in f16x3.  `seg` = option seg_chunks; 0 takes the worse of the two
    automatic periods (2 weight tiles when n_pad > 64, else 3)."""
    slices = k * k * (cin_pad // 16)
    tiles = k * k * -(-cin_pad // 64)
    periods = [seg] if seg > 0 else [2, 3]
    n = max(min(4 * p, slices) + -(-tiles // p) for p in periods) if seg != 1 else 1 + slices
    return n + (3 if npl == 2 else 0)


def stored_rounding(ref, npl):
    """Bar of storing the fp64 tensor `ref`: f16x1 one fp16 ulp of it (np.spacing of its fp16 value: 2^-24 below the
    normal range, inf at 65504, NaN past it), f16x3 the hi / lo split.  A numpy `ref` gives a numpy bar."""
    if isinstance(ref, np.ndarray):
        return stored_rounding(torch.from_numpy(ref.astype(np.float64)), npl).numpy()
    r = ref.abs()
    if npl == 1:
        r16 = r.to(torch.float16).to(torch.float64)
        e = torch.frexp(r16)[1]
        sp = torch.ldexp(torch.ones_like(r16), torch.clamp(e - 1, min=-14) - 10)
        sp = torch.where(r16 == 0, 2.0 ** -24, sp)
        sp = torch.where(r16 == 65504, float("inf"), sp)
        return torch.where(torch.isinf(r16), float("nan"), sp)
    return 2.0 ** -22 * r + 2.0 ** -25


def prelu(h, alpha):
    return torch.where(h > 0, h, col(alpha, h.device) * h)


# The kernels' fp32 constants (epilogue.cuh: kLeakySlope, kSeluScale, kSeluScaleAlpha).
LEAKY = float(np.float32(0.1))
SELU_SCALE = float(np.float32(1.0507009873554805))
SELU_SCALE_ALPHA = float(np.float32(1.7580993408473766))
# act_curve's error in units of 2^-24 |f|: sigmoid 1 / (1 + expf(-z)) (expf within 2 ulp, then the add and the divide),
# tanhf within 2 ulp, selu kSeluScaleAlpha * expm1f(z) (expm1f within 1 ulp, then the product; z > 0 one product)
CURVE_U = {"sigmoid": 6, "tanh": 4, "selu": 3}


def activation(act, z, bar, alpha=None):
    """(f(z), its bar) of an activated layer whose fp32 pre-activation lies within `bar` of the fp64 `z`.  prelu, relu
    and leaky_relu have slope at most 1 and their slope product is one of the epilogue roundings `bar` counts; sigmoid,
    tanh and selu add act_curve's libdevice error and carry `bar` through max |f'| over [z - bar, z + bar].  Sigmoid is
    0 once expf(-z) overflows (z < -88), where f(z) < 2^-126."""
    if act == "prelu":
        return prelu(z, alpha), bar
    if act == "relu":
        return z.clamp_min(0.0), bar
    if act == "leaky_relu":
        return torch.where(z > 0, z, LEAKY * z), bar
    near0 = torch.minimum(torch.maximum(torch.zeros_like(z), z - bar), z + bar)   # where f' peaks on the interval
    floor = 0.0
    if act == "sigmoid":
        v, s0 = torch.sigmoid(z), torch.sigmoid(near0)
        d, floor = s0 * (1 - s0), 2.0 ** -126
    elif act == "tanh":
        v, d = torch.tanh(z), 1 - torch.tanh(near0) ** 2
    elif act == "selu":
        v = torch.where(z < 0, SELU_SCALE_ALPHA * torch.expm1(z), SELU_SCALE * z)
        d = SELU_SCALE_ALPHA * torch.exp(torch.clamp_max(z + bar, 0.0))     # >= kSeluScale once the interval reaches 0
    else:
        raise ValueError(act)
    return v, d * bar + CURVE_U[act] * U24 * (v.abs() + d * bar) + floor


def isolated_layers(eng, cfg, w, x, x2, y, npl, seg, fused, act="prelu", masks=None, keep=1.0, pre=None, device=None,
                    chunk=None):
    """{layer: max err / bar} of one forward whose activations `eng` still holds (see module docstring), for activator
    `act`.  With `masks` ({layer: dropout_mask}, the train step's forward) a kept element's reference is
    f(z) fp32(1 / keep), one more 2^-24 rounding, and a dropped element must be exactly 0.  `pre`, if given, receives
    {activated layer: (fp64 pre-activation z, bar of the GPU's fp32 z)}, or is called as pre(layer, z, bar, images)
    once per slice of images.

    The references are formed on `device` (default: the CPU), `chunk` images at a time (default: all at once).  Images
    are independent, so the slices give the same maxima as one pass.  Each slice fetches the activations it reads and
    keeps only its images of them, so host memory stays at one whole activation at a time."""
    n, h, wd = x.shape[:3]
    f = O.feature_filters(cfg)
    k = cfg.cnn_size
    cps = cfg.nin_filters + cfg.nin_filters2
    ps_out = cfg.pixel_shuffler_filters or cps
    inv_keep = float(np.float32(1.0) / np.float32(keep))
    if isinstance(pre, dict) and chunk is not None and chunk < n:
        raise ValueError("a pre-activation dict holds one slice: pass a callable with chunk")
    out = {}

    def check(name, got, ref, bar, dropped=None):
        ratio = (got - ref).abs() / (bar + 1e-300)     # the floor keeps an exact zero (bar 0) from giving 0 / 0
        if dropped is not None:
            ratio = torch.where(dropped, torch.where(got == 0, 0.0, float("inf")), ratio)
        out[name] = max(out.get(name, 0.0), float(ratio.max()))

    for i0 in range(0, n, chunk or n):
        sl = slice(i0, min(n, i0 + (chunk or n)))

        def plane(name, c, r=1):
            return nchw(eng.get_activation(name, (n, r * h, r * wd, c))[sl], device)

        def tc_layer(a, wq, b, kk, cin_pad):
            """(pre-activation, accumulation + epilogue bar) of one tensor-core layer on the GPU's input `a`."""
            v = conv(a, wq) + col(b, device)
            s = conv(a.abs(), np.abs(wq))
            bar = tc_units(kk, cin_pad, seg, npl) * U23 * s + U23 * (s + col(np.abs(b), device))
            return v, bar

        def activated(scope, z, bar):
            """(stored value, bar, dropped elements or None) of an activated layer from its pre-activation."""
            if callable(pre):
                pre(scope, z, bar, sl)
            elif pre is not None:
                pre[scope] = (z, bar)
            alpha = w["%s/prelu/%s_prelu" % (scope, scope)] if act == "prelu" else None
            v, bar = activation(act, z, bar, alpha)
            if masks is None:
                return v, bar, None
            m = nchw(masks[scope][sl], device)
            v = v * inv_keep
            return v * m, bar * inv_keep + U24 * v.abs(), m == 0

        def store_check(name, got, v, bar, dropped=None):
            check(name, got, v, bar + stored_rounding(v, npl), dropped)

        # CNN1 (fp32 CUDA cores on x)
        a = nchw(x[sl], device)
        w1 = w["CNN1/conv_W"].astype(np.float64)
        s = conv(a.abs(), np.abs(w1))
        b1 = w["CNN1/conv_B"].astype(np.float64)
        v, bar, dropped = activated("CNN1", conv(a, w1) + col(b1, device),
                                    k * k * U24 * s + U23 * (s + col(np.abs(b1), device)))
        feats = [plane("CNN1", f[0])]
        store_check("CNN1", feats[0], v, bar, dropped)
        for i in range(1, cfg.layers):
            sc = "CNN%d" % (i + 1)
            (wq,) = quantise([w[sc + "/conv_W"]], npl)
            v, bar, dropped = activated(sc, *tc_layer(feats[-1], wq, w[sc + "/conv_B"], k, pad16(f[i - 1])))
            feats.append(plane(sc, f[i]))
            store_check(sc, feats[-1], v, bar, dropped)
        # A1 and B1: one packed layer over the concat, one scale
        hc = torch.cat(feats, dim=1)
        del feats
        wa, wb = quantise([w["A1/conv_W"], w["B1/conv_W"]], npl)
        cin_pad = sum(pad16(c) for c in f)
        a1 = plane("A1", cfg.nin_filters)
        b1g = plane("B1", cfg.nin_filters2)
        v, bar, dropped = activated("A1", *tc_layer(hc, wa, w["A1/conv_B"], 1, cin_pad))
        store_check("A1", a1, v, bar, dropped)
        v, bar, dropped = activated("B1", *tc_layer(hc, wb, w["B1/conv_B"], 1, cin_pad))
        store_check("B1", b1g, v, bar, dropped)
        del hc
        (wq,) = quantise([w["B2/conv_W"]], npl)
        v, bar, dropped = activated("B2", *tc_layer(b1g, wq, w["B2/conv_B"], 3, pad16(cfg.nin_filters2)))
        b2 = plane("B2", cfg.nin_filters2)
        store_check("B2", b2, v, bar, dropped)
        # pixel shuffler(s): the last one is fp32 (EPI_D2S_F32) or feeds the fused R-CNN1
        src, cin_pad = torch.cat([b2, a1], dim=1), pad16(cfg.nin_filters2) + pad16(cfg.nin_filters)
        stages = [("Up-PS", "Up-PS/Up-PS_CNN", 2, cps), ("Up-PS2", "Up-PS2/Up-PS2_CNN", 2, ps_out)] if cfg.scale == 4 \
            else [("Up-PS", "Up-PS/Up-PS_CNN", cfg.scale, ps_out)]
        mult = 1
        for si, (name, scope, r, c) in enumerate(stages):
            (wq,) = quantise([w[scope + "/conv_W"]], npl)
            v, bar = tc_layer(src, wq, w[scope + "/conv_B"], k, cin_pad)
            v, bar = O.depth_to_space(v, r), O.depth_to_space(bar, r)
            mult *= r
            if si + 1 < len(stages):            # x4 Up-PS: fp16 planes
                src, cin_pad = plane(name, c, mult), pad16(c)
                store_check(name, src, v, bar)
            elif not fused:
                up = plane(name, c, mult)
                check(name, up, v, bar)
        # R-CNN1 + x2 (fp32)
        wr = w["R-CNN1/conv_W"].astype(np.float64)
        kr = wr.shape[0]
        x2t = nchw(x2[sl], device)
        gpu_y = nchw(y[sl], device)
        if fused:
            yr = conv(v, wr) + x2t
            bar_y = conv(bar, np.abs(wr)) + kr * kr * ps_out * U24 * conv(v.abs(), np.abs(wr)) + U24 * yr.abs()
            check("R-CNN1 (fused)", gpu_y, yr, bar_y)
        else:
            yr = conv(up, wr) + x2t
            bar_y = kr * kr * ps_out * U24 * conv(up.abs(), np.abs(wr)) + U24 * yr.abs()
            check("R-CNN1", gpu_y, yr, bar_y)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("kw,shape,kernels", [c[1:] for c in TC_CASES], ids=[c[0] for c in TC_CASES])
def test_tensor_core_forward_path(kw, shape, kernels, precision):
    """One planner path of the tensor-core graph: the kernels its first (eager) forward reaches, every layer against the
    isolated fp64 reference at the default and the strict promotion periods, fused and unfused, and (f16x3) the output
    against the fp64 oracle and the CUDA-core cross-check.  All bar violations of a case are reported at once."""
    npl = 2 if precision == 0 else 1
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)
    n, h, wd = shape
    s = cfg.scale
    g = np.random.RandomState(n * 1000 + h * 10 + wd)
    x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * wd, 1) * 255).astype(np.float32)
    eng = make_engine(kw, w, precision)
    y, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    assert_kernels_ran(names, [k.format(P=npl) for k in kernels])
    fused = any(k.startswith("conv_last_gather") for k in kernels)
    worst, bad = {}, []
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        for fuse in ((1, 0) if fused else (1,)):
            eng.set_option("fuse_last", fuse)
            y = gpu_forward(eng, x, x2)
            for name, ratio in isolated_layers(eng, cfg, w, x, x2, y, npl, seg, fused and fuse == 1).items():
                worst[name] = max(worst.get(name, 0.0), ratio)
                if not ratio <= 1.0:
                    bad.append(("seg_chunks=%d fuse_last=%d" % (seg, fuse), name, ratio))
    eng.set_option("seg_chunks", 0)
    eng.set_option("fuse_last", 1)
    print("error / bar:", " ".join("%s %.3f" % kv for kv in worst.items()))
    assert not bad, bad
    if npl == 2:
        y64 = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
        y32 = O.Oracle(cfg, w, torch.float32).forward(x, x2)
        y_tc = assert_stress(eng, x, x2, y64, y32)
        eng.set_option("conv_impl", 1)
        y_ref = gpu_forward(eng, x, x2)
        eng.set_option("conv_impl", 0)
        assert np.abs(y_tc - y_ref).max() <= 2e-3
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kw,shape,kernels", [c[1:] for c in DS_CASES], ids=[c[0] for c in DS_CASES])
def test_depthwise_separable_forward_path(kw, shape, kernels):
    """The kernels the forward reached, the output within 1e-3 of the fp64 oracle and every layer at the fp32-level bar
    of check_depthwise_separable_layers (test_gpu_forward.py), on the same inputs; all mismatches reported at once."""
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=4)
    n, h, wd = shape
    s = cfg.scale
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(n, h, wd, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(n, s * h, s * wd, 1, generator=g) * 255).numpy()
    y64, inter = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                         return_intermediates=True)
    eng = make_engine(kw, w)
    y, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    assert_kernels_ran(names, kernels)
    bad = []
    err = float(np.abs(y - y64).max())
    if not err <= TOL:
        bad.append(("output", err))
    for name, ref in inter.items():
        if name == "R-CNN":
            continue
        err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
        if not err <= 2e-6 * max(1.0, np.abs(ref).max()) + 1e-4:
            bad.append((name, err, float(np.abs(ref).max())))
    eng.close()
    assert not bad, bad


INFERENCE_KERNEL = re.compile(r"dcscn::(conv_tc_kernel<\d+, \d+>|conv_first3x3_kernel<false>|conv_first_kernel|"
                              r"conv_last_kernel|conv_last_gather_kernel|conv_last_gather4_kernel|ds_tile_kernel<\d+, \d+>|"
                              r"ds_single_kernel<\d+>|ds_single4_kernel)\(")


def test_every_inference_kernel_has_a_forward_case():
    """Every inference compute kernel in the library (nm -C) is named by a case above, so a new instantiation or kernel
    cannot ship without a forward case that proves it runs and checks what it computes."""
    lib = os.path.join(PKG, "csrc", "libdcscn_b200.so")
    built = set(INFERENCE_KERNEL.findall(subprocess.run(["nm", "-C", lib], check=True, capture_output=True,
                                                        text=True).stdout))
    assert len([k for k in built if k.startswith("conv_tc_kernel<")]) == 14, sorted(built)
    assert len([k for k in built if k.startswith("ds_tile_kernel<")]) == 10, sorted(built)
    named = {k.format(P=p) for c in TC_CASES for k in c[3] for p in (1, 2)} | {k for c in DS_CASES for k in c[3]}
    assert not sorted(built - named), sorted(built - named)
