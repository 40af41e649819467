"""
Depthwise-separable graphs wider than the fp32 CUDA-core kernels (run with `-m gpu` on an H100).  Such a graph runs on
the tensor-core graph's buffers and plans: each k x k separable layer as depthwise_planes_kernel (fp32 FMAs over fp16
hi/lo planes) followed by a 1x1 conv_tc_kernel layer of its pointwise filter, and every other layer with its
depthwise filter folded into a dense one (engine.cu: ds_tile_fits, ds_split, layer_filter).

  * forward parity against the fp64 oracle with the stress bars of test_gpu_forward.py, fused and unfused, at the
    default and strict promotion periods, with a profiler check that the depthwise kernel ran and ds_tile_kernel did not;
  * isolated per-layer bars (f16x3 and f16x1) for every split layer, recomputed in fp64 from the input planes the GPU
    stored: the depthwise step at k^2 2^-24 sum |x| |dw| plus the hi / lo store rounding of u, carried through the
    pointwise layer, which has the 1x1 tc_units bar of test_gpu_forward_paths.py;
  * the shipped depthwise-separable checkpoint still runs on ds_tile_kernel alone;
  * tiled forwards, the self-ensemble and CUDA-graph replays equal the whole-image, eager forward bit for bit;
  * the train step: the dense tensor-core step on composed filters W[t][ci][co] = dw[t][ci] pw[ci][co], with the filter
    gradients mapped back to depthwise_W / pointwise_W, against fp64 autograd, through optimizer steps, 200 steps of
    real patches and the train.py / evaluate.py command lines.
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
from conftest import GOLDEN, MODEL_FLAGS, PKG, load_golden_weights
from test_gpu_forward import SMALL, assert_stress, gpu_forward, make_engine, stress_bound
from test_gpu_forward_paths import U23, U24, conv, nchw, pad16, prelu, quantise, stored_rounding, tc_units
from test_gpu_train import assert_kernels_ran, launched_kernels, oracle_masks, setup

pytestmark = pytest.mark.gpu

DSW = dict(depthwise_separable=True)
CASES = [
    # id, config, (n, h, w)
    ("L8F96-x2", dict(DSW, layers=8, filters=96), (1, 12, 14)),                       # default NIN 64 + 32
    ("x4", dict(SMALL, scale=4, **DSW), (1, 9, 11)),                                  # Up-PS2 at 2x resolution
    ("x3-k5", dict(SMALL, scale=3, cnn_size=5, **DSW), (1, 9, 11)),
    ("x3-k1", dict(SMALL, scale=3, cnn_size=1, **DSW), (1, 9, 11)),                   # B2 stays 3 x 3
    ("nin48", dict(scale=2, layers=3, filters=12, min_filters=6, nin_filters=32, nin_filters2=16,
                   pixel_shuffler_filters=1, **DSW), (2, 7, 9)),                      # CNN layers fit the fp32 kernels
    ("L12-x2", dict(DSW), (1, 8, 10)),                                                # the full default graph
]
DEPTHWISE = "depthwise_planes_kernel"


def inputs(kw, n, h, w, seed=3):
    s = kw.get("scale", 2)
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, h, w, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(n, s * h, s * w, 1, generator=g) * 255).numpy()
    return x, x2


def assert_wide_path(names):
    assert_kernels_ran(names, [DEPTHWISE, "conv_tc_kernel"])
    ds_tile = sorted(n for n in names if "dcscn::ds_" in n)
    assert not ds_tile, ds_tile


@pytest.mark.parametrize("kw,shape", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_wide_forward_matches_oracle(kw, shape):
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)
    x, x2 = inputs(kw, *shape)
    y64, inter = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                         return_intermediates=True)
    y32 = O.Oracle(cfg, w, torch.float32).forward(x, x2)
    eng = make_engine(kw, w)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    assert_wide_path(names)
    assert_stress(eng, x, x2, y64, y32)
    eng.set_option("fuse_last", 0)
    y = gpu_forward(eng, x, x2)
    assert float(np.abs(y - y64).max()) <= max(1.5e-3, stress_bound(y32, y64))
    bad = []
    for name, ref in inter.items():   # the unfused forward materialises every layer, the pixel shufflers included
        if name == "R-CNN":
            continue
        err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
        if not err <= 4e-6 * max(1.0, np.abs(ref).max()) + 1e-4:
            bad.append((name, err, float(np.abs(ref).max())))
    eng.close()
    assert not bad, bad


def depthwise64(a, dw):
    """tf.nn.depthwise_conv2d(SAME), multiplier 1, of an NCHW fp64 tensor with a [k, k, c, 1] filter."""
    k, c = dw.shape[0], dw.shape[2]
    wt = torch.from_numpy(np.ascontiguousarray(dw[:, :, :, 0].transpose(2, 0, 1), dtype=np.float64)).view(c, 1, k, k)
    return torch.nn.functional.conv2d(a, wt, padding=k // 2, groups=c)


@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("case", ["L8F96-x2", "x3-k5", "x4"])
def test_split_layers_isolated(case, precision):
    """Every split layer (CNN2..CNNL, B2, the pixel shufflers) against fp64 recomputed from the GPU's own stored input
    (module docstring)."""
    kw, shape = {c[0]: c[1:] for c in CASES}[case]
    npl = 2 if precision == 0 else 1
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)
    x, x2 = inputs(kw, *shape)
    n, h, wd = shape
    eng = make_engine(kw, w, precision)
    eng.set_option("fuse_last", 0)
    f = O.feature_filters(cfg)
    k = cfg.cnn_size
    worst, bad = {}, []
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        gpu_forward(eng, x, x2)

        def act(name, c):
            return nchw(eng.get_activation(name, (n, h, wd, c)))

        layers = [("CNN%d" % (i + 1), "CNN%d" % i, f[i - 1], f[i], k) for i in range(1, cfg.layers)]
        layers.append(("B2", "B1", cfg.nin_filters2, cfg.nin_filters2, 3))
        for scope, src, cin, cout, kk in layers:
            a = act(src, cin)
            ratio = split_layer_ratio(w, scope, a, kk, pad16(cin), seg, npl, act(scope, cout), True, 1)
            kind = "B2" if scope == "B2" else "CNN"
            worst[kind] = max(worst.get(kind, 0.0), ratio)
            if not ratio <= 1.0:
                bad.append((seg, scope, ratio))
        # the pixel shufflers (fuse_last = 0 materialises the last one in fp32): Up-PS over [B2 | A1], whose u has
        # the [B2 | A1] buffer's pitch, and at x4 Up-PS2 over the 2x-resolution planes Up-PS stored
        cps = cfg.nin_filters + cfg.nin_filters2
        ps_out = cfg.pixel_shuffler_filters or cps
        src = torch.cat([act("B2", cfg.nin_filters2), act("A1", cfg.nin_filters)], dim=1)
        pitch = pad16(cfg.nin_filters2) + pad16(cfg.nin_filters)
        stages = [("Up-PS", "Up-PS/Up-PS_CNN", cps), ("Up-PS2", "Up-PS2/Up-PS2_CNN", ps_out)] if cfg.scale == 4 else \
            [("Up-PS", "Up-PS/Up-PS_CNN", ps_out)]
        r = 2 if cfg.scale == 4 else cfg.scale
        mult = 1
        for si, (name, scope, c) in enumerate(stages):
            mult *= r
            last = si + 1 == len(stages)
            got = nchw(eng.get_activation(name, (n, mult * h, mult * wd, c)))
            ratio = split_layer_ratio(w, scope, src, k, pitch, seg, npl, got, False, r, stored=not last)
            worst[name] = max(worst.get(name, 0.0), ratio)
            if not ratio <= 1.0:
                bad.append((seg, name, ratio))
            src, pitch = got, pad16(c)
    eng.close()
    print("error / bar:", " ".join("%s %.3f" % kv for kv in worst.items()))
    assert not bad, bad


def split_layer_ratio(w, scope, a, kk, cin_pad, seg, npl, got, activated, r, stored=True):
    """max error / bar of one split layer on the GPU's input `a` (module docstring); `r` > 1: a pixel shuffler, its
    output through depth_to_space, stored in fp32 when not `stored`."""
    dw = w[scope + "/depthwise_W"].astype(np.float32).astype(np.float64)
    u = depthwise64(a, dw)
    bar_u = kk * kk * U24 * depthwise64(a.abs(), np.abs(dw)) + torch.from_numpy(stored_rounding(u.numpy(), npl))
    (pq,) = quantise([w[scope + "/pointwise_W"]], npl)
    b = w[scope + "/conv_B"].astype(np.float64)
    bt = torch.from_numpy(np.abs(b)).view(1, -1, 1, 1)
    z = conv(u, pq) + torch.from_numpy(b).view(1, -1, 1, 1)
    s = conv(u.abs() + bar_u, np.abs(pq))
    bar = tc_units(1, cin_pad, seg, npl) * U23 * s + conv(bar_u, np.abs(pq)) + U23 * (s + bt)
    if activated:
        alpha = w["%s/prelu/%s_prelu" % (scope, scope)]
        z = prelu(z, alpha)
        bar = bar * max(1.0, float(np.abs(alpha).max()))
    if r > 1:
        z, bar = O.depth_to_space(z, r), O.depth_to_space(bar, r)
    v = z.numpy()
    bar = bar.numpy() + (stored_rounding(v, npl) if stored else 0.0)
    return float((np.abs(got.numpy() - v) / bar).max())


def test_shipped_checkpoint_keeps_the_fp32_kernels():
    model = "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"
    kw = MODEL_FLAGS[model]
    w = load_golden_weights(model)
    x, x2 = inputs(kw, 2, 24, 20)
    eng = make_engine(kw, w)
    y, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    eng.close()
    assert_kernels_ran(names, ["ds_tile_kernel"])
    assert not [nm for nm in names if DEPTHWISE in nm or "conv_tc_kernel" in nm]
    y64 = O.Oracle(O.OracleConfig(**kw), w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert float(np.abs(y - y64).max()) <= 1e-3


@pytest.mark.parametrize("case", ["L8F96-x2", "x4"])
def test_tiled_ensemble_and_graph_replay_are_bit_identical(case):
    kw, _ = {c[0]: c[1:] for c in CASES}[case]
    s = kw.get("scale", 2)
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=2)
    x, x2 = inputs(kw, 2, 45, 61, seed=5)
    eng = make_engine(kw, w)
    eng.set_option("graph", 0)
    la = eng.launch_count
    y_whole = gpu_forward(eng, x, x2)
    per_forward = eng.launch_count - la
    px_bytes = eng.device_bytes / float(2 * 45 * 61)
    e_whole = eng.forward_ensemble_host(x[0], x2[0], 8)
    eng.set_option("graph", 1)
    xs, x2s = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
    r0, l0 = eng.graph_replays, eng.launch_count
    ys = [eng.forward(xs, x2s).cpu().numpy() for _ in range(4)]       # eager, capture + replay, replays
    assert eng.graph_replays - r0 >= 2
    assert eng.launch_count - l0 == 4 * per_forward
    for y in ys:
        assert np.array_equal(y, y_whole)
    eng.set_option("workspace_mb", -(-int(px_bytes * 3000) >> 20))   # windows of about 3000 LR pixels
    eng.set_option("timing", 1)
    y_tiled = gpu_forward(eng, x, x2)
    assert sum(nm == "tile_stitch" for nm, _ in eng.timings()) >= 2
    eng.set_option("timing", 0)
    e_tiled = eng.forward_ensemble_host(x[0], x2[0], 8)
    eng.close()
    assert np.array_equal(y_tiled, y_whole)
    assert np.array_equal(e_tiled, e_whole)
    assert y_whole.shape == (2, s * 45, s * 61, 1)


def test_timings_name_the_depthwise_launches():
    kw, shape = {c[0]: c[1:] for c in CASES}["x4"]
    cfg = O.OracleConfig(**kw)
    eng = make_engine(kw, O.he_init_weights(cfg, seed=0))
    eng.set_option("timing", 1)
    x, x2 = inputs(kw, *shape)
    gpu_forward(eng, x, x2)
    names = [nm for nm, _ in eng.timings()]
    eng.close()
    split = ["CNN%d" % (i + 1) for i in range(1, cfg.layers)] + ["B2", "Up-PS", "Up-PS2"]
    assert names == ["CNN1"] + sum([["dw:" + nm, nm] for nm in split[:-3]], []) + ["A1+B1"] + \
        sum([["dw:" + nm, nm] for nm in split[-3:]], []) + ["R-CNN1"], names


def test_train_step_updates_reach_the_wide_forward():
    """After a train step the next forward uses the updated weights."""
    kw, _ = {c[0]: c[1:] for c in CASES}["nin48"]
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=1)
    eng = make_engine(kw, w)
    x, x2 = inputs(kw, 4, 12, 12, seed=7)
    y = x2 + np.float32(3.0)
    eng.train_step_host(x, x2, y, 1e-3, 11)
    w_new = {name: eng.get_param(name) for name in w}
    assert any(not np.array_equal(w_new[nm], w[nm]) for nm in w if nm.endswith("pointwise_W"))
    xa, xb = inputs(kw, 1, 10, 13, seed=8)
    got = gpu_forward(eng, xa, xb)
    eng.close()
    ref = O.Oracle(cfg, w_new, torch.float64).forward(xa.astype(np.float64), xb.astype(np.float64))
    assert float(np.abs(got - ref).max()) <= 1e-3


TRAIN_CASES = [
    # id, config, (n, h, w): x2 / x3 / x4 and k = 1, 3, 5
    ("nin48-x2", {c[0]: c[1] for c in CASES}["nin48"], (2, 9, 8)),
    ("x3-k5", {c[0]: c[1] for c in CASES}["x3-k5"], (2, 8, 7)),
    ("x3-k1", {c[0]: c[1] for c in CASES}["x3-k1"], (2, 8, 7)),
    ("x4", {c[0]: c[1] for c in CASES}["x4"], (1, 7, 9)),
]


@pytest.mark.parametrize("kw,shape", [c[1:] for c in TRAIN_CASES], ids=[c[0] for c in TRAIN_CASES])
def test_wide_gradients_match_oracle(kw, shape):
    """Loss and every gradient within 2e-3 of the tensor's max against fp64 autograd with the engine's dropout masks
    (the dense step's bar); the dead conv_W's gradient is exactly its L2 decay."""
    n, h, w = shape
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, w, seed=5)
    seed = 4321
    (loss, mse), names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, ["ds_compose_kernel", "ds_decompose_kernel", "wgrad_tc_kernel"])
    assert not [nm for nm in names if "dcscn::ds_" in nm and "compose" not in nm], names
    masks = oracle_masks(eng, cfg, seed, n, h, w)
    mse_ref, _, grads_ref = O.Oracle(cfg, wts, torch.float64).loss_and_grads(
        x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
    bad = []
    if not mse == pytest.approx(mse_ref, rel=5e-5):
        bad.append(("mse", mse, mse_ref))
    for name, gref in grads_ref.items():
        err = float(np.abs(eng.get_grad(name) - gref).max())
        if not err <= 2e-3 * np.abs(gref).max() + 1e-7:
            bad.append((name, err, float(np.abs(gref).max())))
    for name in wts:
        if name.endswith("conv_W"):
            np.testing.assert_array_equal(eng.get_grad(name), np.float32(cfg.l2_decay) * wts[name].astype(np.float32))
    eng.close()
    assert not bad, bad


@pytest.mark.parametrize("optimizer", ["adam", "gd"])
def test_wide_optimizer_steps_and_forward_follow(optimizer):
    """Three steps against the oracle's clip + update, then the forward sees the updated weights."""
    from helper import engine as E
    kw = {c[0]: c[1] for c in CASES}["x4"]
    n, h, w = 2, 10, 10
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, w, seed=9)
    eng.close()
    eng = E.Engine(E.make_config(dropout_keep=0.8, optimizer=optimizer, **kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    orc = O.Oracle(cfg, wts, torch.float64)
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
    ref = O.Oracle(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(
        x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3


def test_wide_200_steps_raise_set5_psnr_and_precisions_agree(tmp_path):
    """200 steps of real Set14 patches on a wide graph (NIN 32 + 16) take random weights to a usable up-scaler; on the
    trained weights the f16x1 and f16x3 forwards give the same Set5 PSNR within 0.01 dB."""
    import random
    from helper import args as A
    import DCSCN
    random.seed(1234)
    np.random.seed(1234)
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog", "--scale=2", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2",
             "--nin_filters=32", "--nin_filters2=16", "--reconstruct_layers=0", "--pixel_shuffler_filters=1",
             "--depthwise_separable=true", "--self_ensemble=1", "--batch_num=20", "--batch_image_size=32",
             "--build_batch=true", "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14",
             "--batch_dir=" + str(tmp_path / "batch"), "--checkpoint_dir=" + str(tmp_path / "ckpt"),
             "--log_filename=" + str(tmp_path / "log.txt"), "--tf_log_dir=" + str(tmp_path / "tf_log"),
             "--graph_dir=" + str(tmp_path / "graphs"), "--output_dir=" + str(tmp_path / "out")])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.load_datasets(f.data_dir + "/" + f.dataset, f.batch_dir + "/" + f.dataset, f.batch_image_size, f.stride_size)
    m.build_graph()
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    m.init_train_step()
    m.init_epoch_index()
    test_files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    curve = [m.evaluate(test_files)[0]]
    for step in range(200):
        m.build_input_batch()
        m.train_batch()
    curve.append(m.evaluate(test_files)[0])
    print("Set5 PSNR before / after 200 steps:", curve)
    assert np.isfinite(curve).all()
    assert curve[-1] >= curve[0] + 8.0 and curve[-1] >= 28.0, curve
    weights = {name: m.engine.get_param(name) for name in m.engine.param_shapes()}
    psnr = {}
    for prec in (0, 1):
        eng = make_engine(dict(scale=2, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=32,
                               nin_filters2=16, reconstruct_layers=0, pixel_shuffler_filters=1, **DSW), weights, prec)
        ps = []
        for fn in test_files:
            lr_img, bic, true_y = O.build_inputs_for_evaluate(fn, 2)
            y = gpu_forward(eng, lr_img.reshape(1, *lr_img.shape).astype(np.float32),
                            bic.reshape(1, *bic.shape).astype(np.float32))
            ps.append(O.compute_psnr(true_y, y[0], 2))
        eng.close()
        psnr[prec] = float(np.mean(ps))
    assert abs(psnr[0] - psnr[1]) < 0.01, psnr


def test_train_and_evaluate_cli_l8_f96(tmp_path):
    """train.py --depthwise_separable --layers=8 --filters=96 trains a few steps and saves; evaluate.py with the same
    flags loads that checkpoint and prints a PSNR."""
    from helper import tf_bundle
    ckpt = tmp_path / "ckpt"
    common = ["--scale=2", "--layers=8", "--filters=96", "--depthwise_separable=true", "--self_ensemble=1",
              "--test_dataset=set5", "--data_dir=" + os.path.join(GOLDEN, "data"), "--checkpoint_dir=" + str(ckpt),
              "--log_filename=" + str(tmp_path / "log.txt"), "--tf_log_dir=" + str(tmp_path / "tf_log"),
              "--graph_dir=" + str(tmp_path / "graphs"), "--output_dir=" + str(tmp_path / "out")]
    train = [sys.executable, os.path.join(PKG, "train.py"), "--dataset=set5", "--training_images=16", "--batch_num=8",
             "--batch_image_size=16", "--lr_decay_epoch=1", "--lr_decay=0.01", "--end_lr=1e-5",
             "--batch_dir=" + str(tmp_path / "batch")] + common
    r = subprocess.run(train, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    files = glob.glob(str(ckpt / "*.ckpt*"))
    assert files, os.listdir(str(tmp_path))
    name = [fn for fn in files if fn.endswith(".ckpt.index")][0][:-len(".index")] if any(
        fn.endswith(".ckpt.index") for fn in files) else files[0]
    rd = tf_bundle.BundleReader(name)
    assert "CNN2/depthwise_W" in rd.keys() and "CNN2/pointwise_W/Adam" in rd.keys()
    assert np.isfinite(rd.get_tensor("CNN2/pointwise_W")).all()
    ev = [sys.executable, os.path.join(PKG, "evaluate.py"), "--save_results=false"] + common
    r = subprocess.run(ev, cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    log = open(tmp_path / "log.txt").read()
    found = re.findall(r"Model Average \[set5\] PSNR:([0-9.]+)", log)
    assert found and all(np.isfinite(float(v)) for v in found), log
