"""
Scale factors above x4 (--scale=5 to 8) on the H100 (run with `-m gpu`).  x5..x8 run through the same kernels as x2 and
x3: one Up-PS (or Up-TCNN with K = 2s - s%2) into s*s*C columns with a depth_to_space(s) epilogue, the fused R-CNN1
where get_plan's rule allows it, and the s2d / R-CNN1 / Up-PS backward kernels at r = s.  L12 x8 has an Up-PS of
64 * 96 = 6144 columns.

  * forward parity against the fp64 oracle with the stress bars of test_gpu_forward.py (fused and unfused, both
    promotion periods) at x5..x8, full-width L12 and L8 F96 at x8, Up-TCNN at x5 / x8 and depthwise-separable graphs
    narrow and wide at x8, each with a profiler check that only the existing inference kernels ran;
  * the isolated per-layer bars of test_gpu_forward_paths.py (f16x3 and f16x1) for Up-PS and Up-TCNN at x8;
  * tiled forwards, the 8-flip ensemble and CUDA-graph replays bit-identical to the plain forward at x8;
  * every gradient against fp64 autograd at x5 and x8, the isolated per-kernel backward bars of
    test_gpu_backward_paths.py at r = 8, and Adam / gd steps;
  * the crop and patch gathers at x8 bit-identical to the host loader, device evaluation == host evaluation at x8 and
    x5, 200 real-crop steps at x8 and the train.py / evaluate.py command lines with an Sc8 checkpoint.
"""
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from conftest import GOLDEN, MODEL_FLAGS, PKG
from test_gpu_backward_paths import Checker, capture_step, check_step, real_patches, report
from test_gpu_eval import SET5, SET14, check_files
from test_gpu_forward import assert_stress, gpu_forward, make_engine, stress_bound
from test_gpu_forward_paths import INFERENCE_KERNEL, U23, conv, isolated_layers, nchw, pad16, quantise, tc_units
from test_gpu_train import assert_kernels_ran, launched_kernels, oracle_masks
from test_large_scale_cpu import _flags
from test_tiling_cpu import tile_halo

pytestmark = pytest.mark.gpu

PS32 = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
TC = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=32, nin_filters2=16,
          transposed_upsampler=True)
CDS = dict(MODEL_FLAGS["dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"])     # c-DCSCN, depthwise-separable
DSW = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=24, nin_filters2=16,
           depthwise_separable=True)                                            # NIN 40 > 32: the wide path
DS12 = dict(layers=3, filters=10, min_filters=6, filters_decay_gamma=1.5, nin_filters=8, nin_filters2=4,
            pixel_shuffler_filters=0, depthwise_separable=True)                 # narrow, R-CNN1 12 -> 1
FWD_CASES = [
    # id, config, (n, h, w)
    ("x5", dict(PS32, scale=5), (1, 9, 11)),                 # 800 columns, HR width 55: one-pixel gather
    ("x6", dict(PS32, scale=6), (1, 9, 10)),                 # HR width 60: four-pixel gather
    ("x7", dict(PS32, scale=7), (2, 7, 9)),                  # HR width 63
    ("x8", dict(PS32, scale=8), (1, 9, 11)),                 # 2048 columns
    ("L12-x8", dict(scale=8), (1, 8, 10)),                   # 6144 columns
    ("L8F96-x8", dict(scale=8, layers=8, filters=96), (1, 8, 10)),
    ("tcnn-x5", dict(TC, scale=5), (1, 9, 11)),              # K = 9
    ("tcnn-x8", dict(TC, scale=8), (1, 8, 10)),              # K = 16, 3072 columns
    ("ds-narrow-x8", dict(CDS, scale=8), (2, 7, 9)),         # Up-PS 32 -> 64 on ds_tile_kernel
    ("ds-narrow12-x8", dict(DS12, scale=8), (1, 6, 5)),      # Up-PS 12 -> 768
    ("ds-wide-x8", dict(DSW, scale=8), (1, 9, 11)),          # depthwise_planes_kernel + 2560-column pointwise Up-PS
]
DEPTHWISE = "depthwise_planes_kernel"


def oracle_for(kw):
    if kw.get("transposed_upsampler"):
        cfg = T.Config(**kw)
        return cfg, T.random_weights(cfg, seed=0), T.Oracle
    cfg = O.OracleConfig(**kw)
    return cfg, O.he_init_weights(cfg, seed=0), O.Oracle


def inputs(s, n, h, w, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, h, w, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(n, s * h, s * w, 1, generator=g) * 255).numpy()
    return x, x2


def only_inference_kernels(names):
    ours = sorted(n for n in names if "dcscn::" in n)
    assert ours
    other = [n for n in ours if not INFERENCE_KERNEL.search(n) and "dcscn::%s" % DEPTHWISE not in n]
    assert not other, other


def test_scales_outside_2_to_8_are_refused():
    from helper import engine as E
    for s in (1, 9, 0, -2):
        with pytest.raises(E.EngineError, match="2..8"):
            E.Engine(E.make_config(scale=s))
    E.Engine(E.make_config(scale=8)).close()


@pytest.mark.parametrize("kw,shape", [c[1:] for c in FWD_CASES], ids=[c[0] for c in FWD_CASES])
def test_forward_matches_oracle(kw, shape):
    cfg, w, Orc = oracle_for(kw)
    s = cfg.scale
    x, x2 = inputs(s, *shape)
    y64, inter = Orc(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64), return_intermediates=True)
    eng = make_engine(kw, w)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    only_inference_kernels(names)
    narrow_ds = kw.get("depthwise_separable") and kw["nin_filters"] + kw["nin_filters2"] <= 32
    if kw.get("depthwise_separable"):
        assert_kernels_ran(names, ["ds_tile_kernel"] if narrow_ds else [DEPTHWISE, "conv_tc_kernel"])
    else:
        assert_kernels_ran(names, ["conv_tc_kernel"])
    if narrow_ds:       # fp32 CUDA cores: the bars of check_depthwise_separable_layers
        y = gpu_forward(eng, x, x2)
        assert np.abs(y - y64).max() <= 1e-3
        tol = lambda ref: 2e-6 * max(1.0, np.abs(ref).max()) + 1e-4
    else:
        y32 = Orc(cfg, w, torch.float32).forward(x, x2)
        assert_stress(eng, x, x2, y64, y32)
        eng.set_option("fuse_last", 0)
        y = gpu_forward(eng, x, x2)
        assert float(np.abs(y - y64).max()) <= max(1.5e-3, stress_bound(y32, y64))
        tol = lambda ref: 4e-6 * max(1.0, np.abs(ref).max()) + 1e-4
    bad = []
    for name, ref in inter.items():   # the unfused forward materialises every layer, the upsampler included
        if name == "R-CNN":
            continue
        err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
        if not err <= tol(ref):
            bad.append((name, err, float(np.abs(ref).max())))
    eng.close()
    assert not bad, bad


def test_fused_last_layer_follows_the_existing_rule():
    """get_plan fuses R-CNN1 into the Up-PS epilogue for 16-aligned pixel-shuffler outputs up to 128 channels: the
    32- and 96-channel x8 graphs take it, the 40-channel wide DS graph and c-DCSCN (1 channel) do not."""
    for kw, fused in ((dict(PS32, scale=8), True), (dict(scale=8), True), (dict(PS32, scale=5), True),
                      (dict(DSW, scale=8), False), (dict(MODEL_FLAGS["dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32"], scale=8), False)):
        cfg, w, _ = oracle_for(kw)
        x, x2 = inputs(cfg.scale, 1, 8, 8)
        eng = make_engine(kw, w)
        _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
        eng.close()
        assert any("dcscn::conv_last_gather" in n for n in names) == fused, (kw, sorted(n for n in names if "dcscn::" in n))


@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("case", ["x8", "L12-x8"])
def test_up_ps_layers_isolated(case, precision):
    """Every layer of the x8 graph, Up-PS included, against the isolated fp64 reference of test_gpu_forward_paths.py
    at the default and strict promotion periods, fused and unfused."""
    kw, shape = {c[0]: c[1:] for c in FWD_CASES}[case]
    npl = 2 if precision == 0 else 1
    cfg, w, _ = oracle_for(kw)
    x, x2 = inputs(cfg.scale, *shape)
    eng = make_engine(kw, w, precision)
    worst, bad = {}, []
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        for fuse in (1, 0):
            eng.set_option("fuse_last", fuse)
            y = gpu_forward(eng, x, x2)
            for name, ratio in isolated_layers(eng, cfg, w, x, x2, y, npl, seg, fuse == 1).items():
                worst[name] = max(worst.get(name, 0.0), ratio)
                if not ratio <= 1.0:
                    bad.append((seg, fuse, name, ratio))
    eng.close()
    print("error / bar:", " ".join("%s %.3f" % kv for kv in worst.items()))
    assert not bad, bad


@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
def test_up_tcnn_layer_isolated(precision):
    """Up-TCNN at x8 (K = 16) from the [B2 | A1] planes the GPU stored, F quantised as pack_tc_layer does."""
    kw, shape = {c[0]: c[1:] for c in FWD_CASES}["tcnn-x8"]
    npl = 2 if precision == 0 else 1
    cfg, w, _ = oracle_for(kw)
    s = cfg.scale
    x, x2 = inputs(s, *shape)
    n, h, wd = shape
    c = cfg.nin_filters + cfg.nin_filters2
    pitch = pad16(cfg.nin_filters2) + pad16(cfg.nin_filters)
    eng = make_engine(kw, w, precision)
    eng.set_option("fuse_last", 0)
    (fq,) = quantise([T.tconv_filter(w[T.TCONV], s)], npl)
    worst = 0.0
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        gpu_forward(eng, x, x2)
        a = torch.cat([nchw(eng.get_activation("B2", (n, h, wd, cfg.nin_filters2))),
                       nchw(eng.get_activation("A1", (n, h, wd, cfg.nin_filters)))], dim=1)
        z = O.depth_to_space(conv(a, fq), s)
        sabs = O.depth_to_space(conv(a.abs(), np.abs(fq)), s)
        bar = (tc_units(3, pitch, seg, npl) * U23 * sabs + U23 * sabs).numpy()
        got = nchw(eng.get_activation("Up-TCNN", (n, s * h, s * wd, c))).numpy()
        worst = max(worst, float((np.abs(got - z.numpy()) / (bar + 1e-30)).max()))
    eng.close()
    print("Up-TCNN x8 error / bar: %.3f" % worst)
    assert worst <= 1.0


@pytest.mark.parametrize("case", ["x8", "L12-x8", "tcnn-x8", "ds-narrow-x8"])
def test_tiled_ensemble_and_graph_replay_are_bit_identical(case):
    """Tiled forwards (a budget that forces several windows) and the 8-flip ensemble equal the whole-image results bit
    for bit; CUDA-graph replays equal the eager forward; the halo is the formula of test_tiling_cpu.py /
    test_tconv_cpu.py; a tiled forward stays inside its workspace budget."""
    from test_tconv_cpu import tile_halo as tconv_halo
    kw, _ = {c[0]: c[1:] for c in FWD_CASES}[case]
    cfg, w, Orc = oracle_for(kw)
    s = cfg.scale
    n, h, wd = 2, 45, 61
    x, x2 = inputs(s, n, h, wd, seed=5)
    eng = make_engine(kw, w)
    eng.set_option("graph", 0)
    la = eng.launch_count
    y_whole = gpu_forward(eng, x, x2)
    per_forward = eng.launch_count - la
    px_bytes = eng.device_bytes / float(n * h * wd)
    e_whole = eng.forward_ensemble_host(x[0], x2[0], 8)
    if not kw.get("depthwise_separable"):
        eng.set_option("graph", 1)
        xs, x2s = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
        r0, l0 = eng.graph_replays, eng.launch_count
        ys = [eng.forward(xs, x2s).cpu().numpy() for _ in range(4)]
        assert eng.graph_replays - r0 >= 2
        assert eng.launch_count - l0 == 4 * per_forward
        for y in ys:
            assert np.array_equal(y, y_whole)
    assert eng.tile_halo() == (tconv_halo(cfg) if kw.get("transposed_upsampler") else tile_halo(cfg))
    mb = -(-int(px_bytes * 2500) >> 20)
    eng.set_option("workspace_mb", mb)
    eng.set_option("timing", 1)
    y_tiled = gpu_forward(eng, x, x2)
    assert sum(nm == "tile_stitch" for nm, _ in eng.timings()) >= 2
    eng.set_option("timing", 0)
    e_tiled = eng.forward_ensemble_host(x[0], x2[0], 8)
    eng.close()
    assert np.array_equal(y_tiled, y_whole)
    assert np.array_equal(e_tiled, e_whole)
    fresh = make_engine(kw, w)                  # only the windows' workspace and staging: within the budget
    fresh.set_option("workspace_mb", mb)
    assert np.array_equal(gpu_forward(fresh, x, x2), y_whole)
    assert 0 < fresh.device_bytes <= mb << 20, (fresh.device_bytes, mb)
    fresh.close()
    y64 = Orc(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert float(np.abs(y_whole - y64).max()) <= 2e-3


# ------------------------------------------------------------------------------------------------- train step ----
TRAIN = dict(layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
CDS_TRAIN = dict(layers=3, filters=12, min_filters=6, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
                 pixel_shuffler_filters=1, depthwise_separable=True)
GRAD_CASES = []
for _s in (5, 8):
    GRAD_CASES += [
        ("tc-x%d" % _s, dict(TRAIN, scale=_s), (2, 6, 7), 2e-3, ["wgrad_tc_kernel", "last_dgrad_s2d_rows_kernel"]),
        ("tcnn-x%d" % _s, dict(TRAIN, scale=_s, transposed_upsampler=True), (2, 6, 7), 2e-3,
         ["wgrad_tc_kernel", "tconv_grad_gather_kernel"]),
        ("ds-narrow-x%d" % _s, dict(CDS_TRAIN, scale=_s), (2, 6, 7), 2e-4, ["ds_dw_fwd_kernel"]),
        ("ds-wide-x%d" % _s, dict(DSW, scale=_s), (1, 6, 7), 2e-3, ["ds_compose_kernel", "ds_decompose_kernel"]),
    ]


def train_setup(kw, keep, n, h, w, seed=0, optimizer="adam"):
    from helper import engine as E
    cfg, _, Orc = oracle_for(kw)
    src = T.random_weights(cfg, seed=seed) if kw.get("transposed_upsampler") else O.he_init_weights(cfg, seed=seed)
    wts = {k: v.astype(np.float64) for k, v in src.items()}
    eng = E.Engine(E.make_config(dropout_keep=keep, optimizer=optimizer, **kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    g = np.random.RandomState(seed + 1)
    s = cfg.scale
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    return cfg, Orc, wts, eng, x, x2, y


@pytest.mark.parametrize("kw,shape,rel,kernels", [c[1:] for c in GRAD_CASES], ids=[c[0] for c in GRAD_CASES])
def test_gradients_match_oracle(kw, shape, rel, kernels):
    """Loss and every gradient within `rel` of the tensor's max against fp64 autograd with the engine's dropout masks
    (the bars of test_gpu_train.py, test_gpu_tconv.py and test_gpu_ds_wide.py)."""
    n, h, w = shape
    cfg, Orc, wts, eng, x, x2, y = train_setup(kw, 0.8, n, h, w, seed=5)
    seed = 4321
    (loss, mse), names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, kernels)
    masks = oracle_masks(eng, cfg, seed, n, h, w)
    mse_ref, _, grads_ref = Orc(cfg, wts, torch.float64).loss_and_grads(
        x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
    bad = []
    if not mse == pytest.approx(mse_ref, rel=5e-5):
        bad.append(("mse", mse, mse_ref))
    for name, gref in grads_ref.items():
        err = float(np.abs(eng.get_grad(name) - gref).max())
        if not err <= rel * np.abs(gref).max() + 1e-7:
            bad.append((name, err, float(np.abs(gref).max())))
    eng.close()
    assert not bad, bad


def test_backward_kernels_isolated_at_r8():
    """The R-CNN1 filter gradient at HR, last_dgrad_s2d_rows (space_to_depth at r = 8), the Up-PS filter gradient and
    dgrad twin at 64 * 32 columns and every other backward kernel, each against its isolated fp64 reference."""
    from test_gpu_train import setup
    kw = dict(TRAIN, scale=8)
    n, h, wd = 2, 9, 11
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, wd)
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=1234, apply_update=False))
    assert_kernels_ran(names, ["last_wgrad_kernel<9>", "last_dgrad_s2d_rows_kernel", "wgrad_tc_kernel", "loss_kernel",
                               "act_grad8_kernel", "grad_finalize_kernel"])
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 1234, Checker())
    report("x8", chk)
    eng.close()
    assert not chk.bad(), chk.bad()


def test_backward_kernels_isolated_l12_x8_real_patches():
    """Full-width L12 at x8 (Up-PS 96 -> 6144 columns) on Set5 / Set14 patches with y = ground truth."""
    from helper import engine as E
    kw = dict(scale=8)
    cfg = O.OracleConfig(**kw)
    wts = O.he_init_weights(cfg, seed=3)
    eng = E.Engine(E.make_config(dropout_keep=0.8, **kw))
    eng.set_params(wts)
    x, x2, y = real_patches(8, 4, 16, 16, 16)
    capture_step(eng, x, x2, y, 0.8, 99)
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 99, Checker())
    report("L12-x8", chk)
    eng.close()
    assert not chk.bad(), chk.bad()


@pytest.mark.parametrize("case,optimizer", [("tc", "adam"), ("tc", "gd"), ("tcnn", "adam")])
def test_optimizer_steps_follow_oracle(case, optimizer):
    """Three steps against the oracle's clip + TF-Adam / gd (the tolerance rule of test_gpu_train.py), then the
    forward sees the updated weights."""
    kw = dict(TRAIN, scale=8, **({"transposed_upsampler": True} if case == "tcnn" else {}))
    n, h, w = 2, 8, 8
    cfg, Orc, wts, eng, x, x2, y = train_setup(kw, 0.8, n, h, w, seed=9, optimizer=optimizer)
    orc = Orc(cfg, wts, torch.float64)
    m = {k: np.zeros_like(v) for k, v in wts.items()}
    v = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    slack = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    lr = 0.002
    for step in range(1, 4):
        seed = 300 + step
        eng.train_step_host(x, x2, y, lr=lr, seed=seed)
        masks = oracle_masks(eng, cfg, seed, n, h, w)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8,
                                         masks=masks)
        clipped, _ = orc.clip_by_global_norm(grads)
        if optimizer == "adam":
            orc.adam_step(clipped, m, v, step, lr)
        else:
            for name in orc.w:
                orc.w[name] = orc.w[name] - lr * clipped[name]
        for name in wts:
            delta = 2e-3 * np.abs(grads[name]).max()
            slack[name] += np.minimum(2.0, 3.0 * delta / (np.abs(grads[name]) + 1e-300)) if optimizer == "adam" else delta
            tol = 2e-3 * lr * step + lr * slack[name]
            got = eng.get_param(name)
            assert (np.abs(got - orc.w[name]) <= tol).all(), (step, name, float((np.abs(got - orc.w[name]) - tol).max()))
    yy = eng.forward_host(x, x2)
    eng.close()
    ref = Orc(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(
        x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3


# ------------------------------------------------------------------------------------------------------- data ----
def test_crop_gather_equals_the_host_loader_at_x8():
    from test_gpu_dynamic_data import dynamic_set, engine, host_and_crops
    ds = dynamic_set("set14", 8, 16)                          # 128 x 128 crops, 1/8 down: 33-tap windows
    eng = engine(scale=8)
    eng.set_image_store(ds.decoded_images())
    for max_value in (255.0, 1.0):
        crops, host = host_and_crops(ds, 24, seed=0, max_value=max_value)
        assert {c[3] for c in crops} == {0, 1}
        assert any(ds.filenames[c[0]].endswith("img_003.png") for c in crops)     # mode 'L' beside RGB in one batch
        for got, want in zip(eng.gather_crops(crops, 16, max_value=max_value), host):
            np.testing.assert_array_equal(got, want)
    eng.close()


def test_patch_gather_equals_the_host_loader_at_x8():
    from helper import engine as E
    from test_gpu_data import KW, build_set, host_batch
    ds = build_set(8, 8)
    eng = E.Engine(E.make_config(dropout_keep=1.0, **dict(KW, scale=8)))
    eng.set_patch_store(ds.input_images, ds.input_interpolated_images, ds.true_images)
    idx = np.random.RandomState(0).randint(0, ds.count, size=13)
    for got, want in zip(eng.gather_patches(idx), host_batch(ds, idx)):
        np.testing.assert_array_equal(got, want)
    eng.close()


@pytest.mark.parametrize("ds_graph", [False, True], ids=["tensor_core", "depthwise_separable"])
def test_crop_step_equals_the_host_buffer_step_at_x8(ds_graph):
    from test_gpu_dynamic_data import KW, dynamic_set, engine, host_and_crops
    kw = dict(CDS, scale=8) if ds_graph else dict(scale=8)
    size = 8
    ds = dynamic_set("set14", 8, size)
    crops, _ = host_and_crops(ds, 8, seed=3, max_value=255.0)
    w = O.he_init_weights(O.OracleConfig(**dict(KW, **kw)), seed=4)
    out = []
    for mode in ("host", "crops"):
        eng = engine(dropout_keep=0.8, **kw)
        eng.set_params(w)
        eng.set_image_store(ds.decoded_images())
        if mode == "host":
            x, x2, y = eng.gather_crops(crops, size)
            res = eng.train_step_host(x, x2, y, lr=1e-3, seed=5)
        else:
            res = eng.train_step_crops(crops, size, lr=1e-3, seed=5)
        names = [nm for nm in eng.param_shapes() if nm.endswith("conv_W")][:3]
        out.append((res, {nm: eng.get_param(nm) for nm in names}))
        eng.close()
    assert out[0][0] == out[1][0]
    for nm in out[0][1]:
        np.testing.assert_allclose(out[0][1][nm], out[1][1][nm], rtol=0, atol=2e-6)


# ------------------------------------------------------------------------------------------------- evaluation ----
def untrained_model(tmp_path, argv):
    """A SuperResolution at its initial (He) weights: no checkpoint exists above x4."""
    import DCSCN
    f = _flags(tmp_path, argv)
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.build_graph()
    m.build_summary_saver()
    m.init_all_variables()
    return m


@pytest.mark.parametrize("scale", [8, 5])
def test_device_evaluation_equals_host(tmp_path, scale):
    m = untrained_model(tmp_path, ["--scale=%d" % scale])
    assert m._device_evaluation() and m.psnr_calc_border_size == scale
    for ensemble in (1, 8):
        m.self_ensemble = ensemble
        check_files(m, SET5 + SET14)         # Set14 img_003 is mode 'L'
    check_files(m, SET14, bicubic=True)


def test_device_evaluation_of_small_images_at_x8(tmp_path):
    """Images a few LR pixels tall after alignment, SSIM with fewer than 11 rows left, and nothing left at all."""
    from PIL import Image
    g = np.random.RandomState(8)
    files = []
    for name, mode, shape in (("rgb", "RGB", (29, 53, 3)), ("gray", "L", (41, 35)), ("tiny", "RGB", (17, 70, 3)),
                              ("tall", "RGB", (90, 24, 3))):
        path = str(tmp_path / (name + ".png"))
        Image.fromarray(g.randint(0, 256, shape).astype(np.uint8), mode).save(path)
        files.append(path)
    m = untrained_model(tmp_path, ["--scale=8"])
    for ensemble in (1, 8):
        m.self_ensemble = ensemble
        with np.errstate(all="ignore"):
            check_files(m, files)
    with np.errstate(all="ignore"):
        got = m.do_for_evaluate(files[2])             # 16 x 64 aligned, a border of 8: nothing left
    assert np.isnan(got[0]) and np.isnan(got[1])


# ------------------------------------------------------------------------------------------------- end to end ----
def test_200_steps_raise_set5_psnr_at_x8(tmp_path):
    """200 steps of random Set14 crops (8 x 8 LR, 64 x 64 HR) from He-initialised weights.  No PSNR target is fixed at
    x8; the start and end values are printed."""
    import random
    import DCSCN
    random.seed(1234)
    np.random.seed(1234)
    f = _flags(tmp_path, ["--scale=8", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2",
                          "--nin_filters=24", "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1",
                          "--self_ensemble=1", "--batch_num=20", "--batch_image_size=8",
                          "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14"])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.load_dynamic_datasets(f.data_dir + "/" + f.dataset, f.batch_image_size)
    m.build_graph()
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    m.init_train_step()
    m.init_epoch_index()
    assert m.batch_crops is not None
    test_files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    curve = [m.evaluate(test_files)[0]]
    for step in range(200):
        m.build_input_batch()
        m.train_batch()
    curve.append(m.evaluate(test_files)[0])
    print("x8 Set5 PSNR before / after 200 steps: %.3f / %.3f" % tuple(curve))
    assert np.isfinite(curve).all()
    assert curve[-1] > curve[0], curve


def test_train_and_evaluate_cli_at_x8(tmp_path):
    """train.py --scale=8 trains a few steps and saves an Sc8 checkpoint with the reference's variable set;
    evaluate.py --scale=8 with the same flags loads it."""
    from helper import tf_bundle
    ckpt = tmp_path / "ckpt"
    common = ["--scale=8", "--layers=4", "--filters=32", "--min_filters=16", "--self_ensemble=1", "--test_dataset=set5",
              "--data_dir=" + os.path.join(GOLDEN, "data"), "--checkpoint_dir=" + str(ckpt),
              "--log_filename=" + str(tmp_path / "log.txt"), "--tf_log_dir=" + str(tmp_path / "tf_log"),
              "--graph_dir=" + str(tmp_path / "graphs"), "--output_dir=" + str(tmp_path / "out")]
    train = [sys.executable, os.path.join(PKG, "train.py"), "--dataset=set5", "--training_images=16", "--batch_num=8",
             "--batch_image_size=8", "--lr_decay_epoch=1", "--lr_decay=0.01", "--end_lr=1e-5",
             "--batch_dir=" + str(tmp_path / "batch")] + common
    r = subprocess.run(train, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    index = glob.glob(str(ckpt / "*.ckpt.index"))
    assert index and "_Sc8_" in os.path.basename(index[0]), os.listdir(str(ckpt))
    rd = tf_bundle.BundleReader(index[0][:-len(".index")])
    cfg = O.OracleConfig(scale=8, layers=4, filters=32, min_filters=16)
    names = {nm for scope, k, cin, cout, bias, act in O.layer_table(cfg) for nm in
             [scope + "/conv_W"] + ([scope + "/conv_B"] if bias else []) +
             (["%s/prelu/%s_prelu" % (scope, scope.split("/")[-1])] if act else [])}
    assert names <= set(rd.keys()), sorted(names - set(rd.keys()))
    assert rd.get_tensor("Up-PS/Up-PS_CNN/conv_W").shape == (3, 3, 96, 64 * 96)
    assert not any(k.startswith("Up-PS2") for k in rd.keys())
    ev = [sys.executable, os.path.join(PKG, "evaluate.py"), "--save_results=false"] + common
    r = subprocess.run(ev, cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    found = re.findall(r"Model Average \[set5\] PSNR:([0-9.]+)", open(tmp_path / "log.txt").read())
    assert found and all(np.isfinite(float(v)) for v in found)
