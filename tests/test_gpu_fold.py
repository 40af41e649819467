"""The last upsampler folded with R-CNN1 (engine.cu build_fold, EPI_D2S_TAPS, train.cuh fold_kernel) on the GPU.

Where get_plan fuses R-CNN1 into the last depth_to_space layer and the operands are f16x3, that layer runs with the
folded filter W' (s*s*9 columns) and writes one set of tap planes, served by get_activation("R-CNN1/taps"):
  * the folded launch in isolation: recomputed in fp64 from the GPU's own input to it with W' folded as the engine does
    (tests/test_fold_cpu.py pins that rounding) and quantised as pack_tc_layer does, at the tensor-core bar of
    test_gpu_forward_paths.py, then the gather + x2 (no R-CNN1 reduction term: the reduction is in the weights);
  * the shipped L12 x2 / x4 checkpoints against the fp64 oracle at the stress bars of test_gpu_forward.py;
  * the c-DCSCN checkpoints (one pixel-shuffler channel) are not fused, so not folded; f16x1 keeps EPI_D2S_RDOT;
  * after optimizer steps the device re-folds from the master weights: bit-identical to a fresh host fold and pack."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcscn_oracle as O
import tconv_oracle as T
from conftest import MODEL_FLAGS, load_golden_weights
from test_fold_cpu import fold32
from test_gpu_forward import assert_stress, gpu_forward, make_engine
from test_gpu_forward_paths import U23, U24, col, conv, nchw, pad16, quantise, tc_units
from test_gpu_train import CDCSCN, SMALL, SMALL3, SMALL4, assert_kernels_ran, launched_kernels, setup

pytestmark = pytest.mark.gpu

L12 = {2: "dcscn_L12_F196to48_NIN_A64_PS_R1F32", 4: "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"}


def noise(s, n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, h, w, 1, generator=g) * 255).numpy(), (torch.rand(n, s * h, s * w, 1, generator=g) * 255).numpy()


def tap_planes(eng, parts, n, hr_h, hr_w):
    return eng.get_activation("R-CNN1/taps", (parts, 9, n, hr_h, hr_w))


def gather9(v):
    """conv_last_gather of tap planes [9, n, H, W] (a torch tensor, on its device): the sum over taps t of plane t at
    the pixel shifted by (t / 3 - 1, t % 3 - 1), zero outside."""
    y = torch.zeros(v.shape[1:], dtype=v.dtype, device=v.device)
    hr_h, hr_w = v.shape[2:]
    p = F.pad(v, (1, 1, 1, 1))
    for t in range(9):
        dy, dx = t // 3 - 1, t % 3 - 1
        y += p[t, :, 1 + dy:1 + dy + hr_h, 1 + dx:1 + dx + hr_w]
    return y


def folded_filter(cfg, w):
    """(W' quantised as pack_tc_layer packs it in f16x3, b') of the last upsampler folded with R-CNN1 (build_fold)."""
    scope = "Up-PS2/Up-PS2_CNN" if cfg.scale == 4 else "Up-PS/Up-PS_CNN"
    wf, bf = fold32(w[scope + "/conv_W"], w[scope + "/conv_B"], w["R-CNN1/conv_W"], cfg.pixel_shuffler_filters or
                    cfg.nin_filters + cfg.nin_filters2)
    (wq,) = quantise([wf], 2)
    return wq, bf


def folded_launch_ratios(eng, cfg, folded, x2, y, seg, device=None, chunk=None):
    """{"taps": max err / bar, "y": max err / bar} of a folded forward whose activations `eng` still holds: the tap
    planes against conv(input, W') + b' in fp64 from the GPU's own input to the folded launch (`folded` =
    folded_filter(cfg, w)), at the tensor-core bar of test_gpu_forward_paths.py, and y against their gather + x2.
    Formed on `device`, `chunk` images at a time (default: all at once)."""
    wq, bf = folded
    n, hr_h, hr_w = y.shape[:3]
    r = 2 if cfg.scale == 4 else cfg.scale          # x4: the 2x second stage
    hh, ww = hr_h // r, hr_w // r                   # the folded launch's pixel grid
    h, wd = hr_h // cfg.scale, hr_w // cfg.scale
    cps = cfg.nin_filters + cfg.nin_filters2
    if cfg.scale == 4:
        srcs, cin_pad = [("Up-PS", (n, hh, ww, cps))], pad16(cps)
    else:
        srcs = [("B2", (n, h, wd, cfg.nin_filters2)), ("A1", (n, h, wd, cfg.nin_filters))]
        cin_pad = pad16(cfg.nin_filters2) + pad16(cfg.nin_filters)
    src = [eng.get_activation(name, shape) for name, shape in srcs]
    taps = tap_planes(eng, 1, n, hr_h, hr_w)[0]
    bfc = col(bf, device)
    out = {"taps": 0.0, "y": 0.0}
    for i0 in range(0, n, chunk or n):
        sl = slice(i0, min(n, i0 + (chunk or n)))
        m = sl.stop - sl.start
        a = torch.cat([nchw(p[sl], device) for p in src], dim=1)
        s_abs = conv(a.abs(), np.abs(wq))
        bar = tc_units(3, cin_pad, seg, 2) * U23 * s_abs + U23 * (s_abs + bfc.abs())
        v = conv(a, wq) + bfc

        def planes(t):   # [m, s*s*9, hh, ww] -> tap planes [9, m, r*hh, r*ww] (EPI_D2S_TAPS)
            return t.reshape(m, r, r, 9, hh, ww).permute(3, 0, 4, 1, 5, 2).reshape(9, m, r * hh, r * ww)
        got = torch.from_numpy(np.ascontiguousarray(taps[:, sl], dtype=np.float64)).to(device)
        out["taps"] = max(out["taps"], float(((got - planes(v)).abs() / planes(bar)).max()))
        # the gather + x2 of the reference planes: their bar carried through, plus the gather's ten fp32 adds
        x2d = torch.from_numpy(np.ascontiguousarray(x2[sl, ..., 0], dtype=np.float64)).to(device)
        y_ref = gather9(planes(v)) + x2d
        bar_y = gather9(planes(bar)) + 10 * U24 * (gather9(planes(v).abs()) + x2d.abs())
        got_y = torch.from_numpy(np.ascontiguousarray(y[sl, ..., 0], dtype=np.float64)).to(device)
        out["y"] = max(out["y"], float(((got_y - y_ref).abs() / bar_y).max()))
    return out


@pytest.mark.parametrize("scale", [2, 4])
def test_folded_launch_isolated(scale):
    """L12 checkpoint (C = 96: the unfolded epilogue writes two partial sets there).  The tap planes against
    conv(input, quantised W') + b' in fp64, and y against their gather + x2, at both promotion periods."""
    model = L12[scale]
    kw = MODEL_FLAGS[model]
    cfg = O.OracleConfig(**kw)
    w = load_golden_weights(model)
    n, h, wd = 2, 13, 17
    x, x2 = noise(scale, n, h, wd, seed=5)
    eng = make_engine(kw, w)
    folded = folded_filter(cfg, w)
    bad = []
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        y = gpu_forward(eng, x, x2)
        ratios = folded_launch_ratios(eng, cfg, folded, x2, y, seg)
        bad += [(name, seg, ratio) for name, ratio in ratios.items() if not ratio <= 1.0]
        print("x%d seg_chunks=%d: taps error / bar %.3f, y error / bar %.3f" % (scale, seg, ratios["taps"], ratios["y"]))
    eng.close()
    assert not bad, bad


@pytest.mark.parametrize("scale", [2, 4])
def test_checkpoints_against_oracle(scale):
    """The shipped L12 checkpoints on uniform-noise tiles, folded, at the stress bars; the fold ran."""
    model = L12[scale]
    kw = MODEL_FLAGS[model]
    cfg = O.OracleConfig(**kw)
    w = load_golden_weights(model)
    n, h, wd = 2, 40, 40
    x, x2 = noise(scale, n, h, wd, seed=1)
    y64 = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    y32 = O.Oracle(cfg, w, torch.float32).forward(x, x2)
    eng = make_engine(kw, w)
    y = assert_stress(eng, x, x2, y64, y32)
    print("x%d: max |y - oracle(fp64)| = %.3e" % (scale, float(np.abs(y - y64).max())))
    assert np.array_equal(gpu_forward(eng, x, x2), y)   # (an option change drops the plans: run the forward again)
    tap_planes(eng, 1, n, scale * h, scale * wd)      # one partial set: the folded launch ran
    eng.close()


@pytest.mark.parametrize("scale", [2, 3, 4])
def test_cdcscn_checkpoints_are_not_folded(scale):
    """pixel_shuffler_filters = 1: R-CNN1 reads one channel, get_plan does not fuse it, so nothing is folded."""
    from helper import engine as E
    model = CDCSCN[scale]
    kw = MODEL_FLAGS[model]
    w = load_golden_weights(model)
    x, x2 = noise(scale, 1, 12, 16)
    eng = make_engine(kw, w)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    assert_kernels_ran(names, ["conv_last_kernel"])
    assert not any("dcscn::conv_last_gather" in nm for nm in names)
    with pytest.raises(E.EngineError):
        tap_planes(eng, 1, 1, 12 * scale, 16 * scale)
    eng.close()


def test_f16x1_keeps_the_partial_sets():
    """f16x1 is each layer on its own fp16 weights: the L12 x2 forward still writes EPI_D2S_RDOT's two partial sets."""
    model = L12[2]
    w = load_golden_weights(model)
    x, x2 = noise(2, 1, 12, 16)
    eng = make_engine(MODEL_FLAGS[model], w, precision=1)
    gpu_forward(eng, x, x2)
    assert tap_planes(eng, 2, 1, 24, 32).shape == (2, 9, 1, 24, 32)
    eng.close()


TCONV = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=32, nin_filters2=16,
             transposed_upsampler=True, scale=2)
REFRESH = [("x2", SMALL), ("x3", SMALL3), ("x4", SMALL4), ("tconv-x2", TCONV),
           ("ds-wide-L8F96", dict(depthwise_separable=True, layers=8, filters=96))]


@pytest.mark.parametrize("kw", [c[1] for c in REFRESH], ids=[c[0] for c in REFRESH])
def test_device_refold_equals_host_fold(kw):
    """Four optimizer steps re-fold on the device after each update; a fresh training engine given the same weights
    folds and packs on the host.  Both forwards, and their tap planes, are bit-identical."""
    from helper import engine as E
    n, h, wd = 2, 12, 14
    if kw.get("transposed_upsampler"):
        cfg = T.Config(**kw)
        wts = T.random_weights(cfg, seed=3)
        eng = E.Engine(E.make_config(dropout_keep=0.8, **kw))
        eng.set_params(wts)
        g = np.random.RandomState(4)
        x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
        x2 = (g.rand(n, 2 * h, 2 * wd, 1) * 255).astype(np.float32)
        y = np.clip(x2 + g.randn(*x2.shape) * 10, 0, 255).astype(np.float32)
    else:
        cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, wd, seed=3)
    s = cfg.scale
    for i in range(4):
        eng.train_step_host(x, x2, y, lr=0.01, seed=50 + i)
    y_dev = eng.forward_host(x, x2)
    v_dev = tap_planes(eng, 1, n, s * h, s * wd)
    params = {nm: eng.get_param(nm) for nm in wts}
    assert any(np.abs(params[nm] - wts[nm]).max() > 1e-3 for nm in wts)      # the weights did move
    fresh = E.Engine(E.make_config(dropout_keep=0.8, **kw))
    fresh.set_params(params)
    # a step without update makes the fresh handle a training one too: a wide depthwise-separable graph then packs its
    # composed k x k filters, as the trained handle does, instead of separate depthwise and pointwise launches
    fresh.train_step_host(x, x2, y, lr=0.01, seed=99, apply_update=False)
    y_host = fresh.forward_host(x, x2)
    v_host = tap_planes(fresh, 1, n, s * h, s * wd)
    eng.close()
    fresh.close()
    assert np.array_equal(v_dev, v_host), float(np.abs(v_dev - v_host).max())
    assert np.array_equal(y_dev, y_host), float(np.abs(y_dev - y_host).max())
